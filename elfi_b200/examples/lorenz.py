"""Lorenz forecast model (mirror of elfi/examples/lorenz.py): the Lorenz 96 ring of n_obs = 40
variables with closure parameters theta1, theta2 and AR(1) stochastic forcing (Wilks 2005), integrated
by RK4 over n_timestep = 160 steps, observed through six summaries (Hakkarainen et al. 2012).

The host path (forecast_lorenz, get_model) consumes the batch's RandomState exactly as the reference
does, so it reproduces the reference's draws, and keeps its quirks: only the default initial state and
n_obs = 40 run (an ndarray initial_state raises ValueError, a list AttributeError, another n_obs
ValueError), and phi > 1 gives NaN rows.  get_device_model is the same task in throughput mode: the
stock priors drawn on the device (DeviceModelPrior), the simulator with its summaries fused on the
device (Philox streams; statistical parity with the host path).

mean, var, cov, xcov and autocov take host arrays (the reference's NumPy code), device tensors
(ops.lorenz_summaries) and the lazy output of the device simulator (the summaries computed in the
simulator); all forms give the same bits."""
from functools import partial

import numpy as np
import scipy.stats as ss
import torch

from .. import device as dev
from .. import model as em
from .. import ops
from ..priors import DeviceModelPrior
from ..throughput import LazySimulation, batch_columns, batch_key

# the state at time 0 of the task (lorenz.py:129-139), one value per variable of the ring
INITIAL_STATE = np.array([
    2.40711741e-01, 4.75597337e+00, 1.19145654e+01, 1.31324866e+00, 2.82675744e+00,
    3.96016971e+00, 2.10479504e+00, 5.47742826e+00, 5.42519447e+00, -1.45166074e+00,
    2.01991521e+00, 3.93873313e+00, 8.22837848e+00, 4.89401702e+00, -5.66278973e+00,
    1.58617220e+00, -1.23849251e+00, -6.04649288e-01, 6.04132264e+00, 7.47588536e+00,
    1.82761402e+00, 3.19209639e+00, -7.58539653e-02, -6.00928508e-03, 4.52902964e-01,
    3.22063602e+00, 7.18613523e+00, 2.39210634e+00, -2.65743666e+00, 2.32046235e-01,
    1.28079141e+00, 4.23344286e+00, 6.94213238e+00, -1.15939497e+00, -5.23037351e-01,
    1.54618811e+00, 1.77863869e+00, 3.30139201e+00, 7.47769309e+00, -3.91312909e-01])
INITIAL_STATE.setflags(write=False)


def _lorenz_ode(y, params):
    """dy/dt of the ring (lorenz.py:18-55) for y (batch, n_obs); params = (eta, theta1, theta2, f)."""
    eta, theta1, theta2, f = params
    g = theta1 + y * theta2
    # variable k couples to k - 2, k - 1 and k + 1 cyclically; the reference writes the columns
    # 0, 1, 2..-2 and -1 separately, which gives the same terms in the same order
    ym2 = np.roll(y, 2, axis=1)
    ym1 = np.roll(y, 1, axis=1)
    yp1 = np.roll(y, -1, axis=1)
    return -ym2 * ym1 + ym1 * yp1 - y + f - g + eta


def runge_kutta_ode_solver(ode, time_step, y, params):
    """One classical RK4 step (lorenz.py:58-91)."""
    k1 = time_step * ode(y, params)
    k2 = time_step * ode(y + k1 / 2, params)
    k3 = time_step * ode(y + k2 / 2, params)
    k4 = time_step * ode(y + k3, params)
    return y + (k1 + 2 * k2 + 2 * k3 + k4) / 6


def forecast_lorenz(theta1=None, theta2=None, f=10., phi=0.984, n_obs=40, n_timestep=160,
                    batch_size=1, initial_state=None, random_state=None, total_duration=4):
    """The stochastic Lorenz 96 forecast (lorenz.py:94-163): (batch_size, n_timestep, n_obs), row 0
    the initial state, then per step n_obs new normals per row, eta = phi eta + e sqrt(1 - phi^2)
    and one RK4 step of length total_duration / n_timestep."""
    if not initial_state:
        initial_state = np.tile(INITIAL_STATE, (batch_size, 1))

    y = initial_state
    eta = 0

    theta1 = np.asarray(theta1).reshape(-1, 1)
    theta2 = np.asarray(theta2).reshape(-1, 1)

    time_step = total_duration / n_timestep

    random_state = random_state or np.random

    time_series = np.empty(shape=(batch_size, n_timestep, n_obs))
    time_series[:, 0, :] = y

    for i in range(1, n_timestep):
        e = random_state.normal(0, 1, y.shape)
        eta = phi * eta + e * np.sqrt(1 - pow(phi, 2))
        y = runge_kutta_ode_solver(_lorenz_ode, time_step, y, (eta, theta1, theta2, f))
        time_series[:, i, :] = y

    return time_series


# ---------------------------------------------------------------------------- summaries
def _summary(x, col):
    """Column col of the six summaries for lazy simulator output or device data; None for host data."""
    if isinstance(x, LazySimulation):
        return x.summaries()[:, col]
    if dev.is_device_array(x):
        return ops.lorenz_summaries(x)[:, col]
    return None


def mean(x):
    """np.mean(x, axis=(1, 2)), the summary 'Mean' (lorenz.py:231-244)."""
    s = _summary(x, 0)
    return np.mean(x, axis=(1, 2)) if s is None else s


def var(x):
    """The mean over space of np.var over time, the summary 'Var' (lorenz.py:247-260)."""
    s = _summary(x, 1)
    return np.mean(np.var(x, axis=1), axis=1) if s is None else s


def autocov(x):
    """The mean over time and space of the lag-1 autocovariance terms, 'Autocov' (lorenz.py:303-320)."""
    s = _summary(x, 2)
    if s is not None:
        return s
    return np.mean((x[:, :-1, :] - np.mean(x[:, :-1, :], keepdims=True, axis=1))
                   * (x[:, 1:, :] - np.mean(x[:, 1:, :], keepdims=True, axis=1)),
                   axis=(1, 2))


def cov(x):
    """The mean over space of the covariance of Y_k with Y_{k+1} over time, 'Cov' (lorenz.py:263-279)."""
    s = _summary(x, 3)
    if s is not None:
        return s
    x_next = np.roll(x, -1, axis=2)
    return np.mean(np.mean((x - np.mean(x, keepdims=True, axis=1))
                           * (x_next - np.mean(x_next, keepdims=True, axis=1)),
                           axis=1), axis=1)


def xcov(x, prev=True):
    """Cross-covariance of Y_k with its previous (prev=True, 'CrosscovPrev') or next neighbour one step
    later (lorenz.py:282-300)."""
    s = _summary(x, 4 if prev else 5)
    if s is not None:
        return s
    x_lag = np.roll(x, 1, axis=2) if prev else np.roll(x, -1, axis=2)
    return np.mean((x[:, :-1, :] - np.mean(x[:, :-1, :], keepdims=True, axis=1))
                   * (x_lag[:, 1:, :] - np.mean(x_lag[:, 1:, :], keepdims=True, axis=1)),
                   axis=(1, 2))


def _graph(m, simulator, y_obs):
    """Priors, simulator, summaries and discrepancy of lorenz.py:205-226."""
    em.Prior(ss.uniform, 0.5, 3., model=m, name='theta1')
    em.Prior(ss.uniform, 0, 0.3, model=m, name='theta2')
    em.Simulator(simulator, m['theta1'], m['theta2'], observed=y_obs, name='Lorenz')
    sumstats = [em.Summary(mean, m['Lorenz'], name='Mean'),
                em.Summary(var, m['Lorenz'], name='Var'),
                em.Summary(autocov, m['Lorenz'], name='Autocov'),
                em.Summary(cov, m['Lorenz'], name='Cov'),
                em.Summary(xcov, m['Lorenz'], True, name='CrosscovPrev'),
                em.Summary(xcov, m['Lorenz'], False, name='CrosscovNext')]
    em.Distance('euclidean', *sumstats, name='d')
    return m


def _observed(true_params, seed_obs, initial_state, n_obs, f, phi, total_duration):
    if not true_params:
        true_params = [2.0, 0.1]
    simulator = partial(forecast_lorenz, initial_state=initial_state, f=f, n_obs=n_obs, phi=phi,
                        total_duration=total_duration)
    return simulator(*true_params, random_state=np.random.RandomState(seed_obs))


def get_model(true_params=None, seed_obs=None, initial_state=None, n_obs=40, f=10., phi=0.984,
              total_duration=4):
    """The Lorenz inference task of lorenz.py:166-228: uniform priors on theta1 (0.5, 3.5) and
    theta2 (0, 0.3), the simulator 'Lorenz', the six summaries and the Euclidean distance."""
    simulator = partial(forecast_lorenz, initial_state=initial_state, f=f, n_obs=n_obs, phi=phi,
                        total_duration=total_duration)
    y_obs = _observed(true_params, seed_obs, initial_state, n_obs, f, phi, total_duration)
    return _graph(em.new_model(), simulator, y_obs)


# ---------------------------------------------------------------------------- throughput mode
def lorenz_device(theta1, theta2, initial_state=INITIAL_STATE, n_timestep=160, f=10., phi=0.984,
                  total_duration=4, batch_size=1, random_state=None):
    """Device twin of forecast_lorenz; returns a LazySimulation of shape (batch_size, n_timestep,
    n_obs) whose six summaries are computed in the simulator kernel."""
    P = torch.stack(batch_columns((theta1, theta2), batch_size), dim=1)
    key = batch_key(random_state)
    kw = dict(initial_state=initial_state, n_timestep=n_timestep, f=f, phi=phi,
              total_duration=total_duration)
    return LazySimulation(
        (int(P.shape[0]), int(n_timestep), len(initial_state)),
        lambda kind: ops.sim_lorenz(P, seed=key, **kw)[1],
        lambda: ops.sim_lorenz(P, seed=key, want_data=True, want_summaries=False, **kw)[0])


def get_device_model(true_params=None, seed_obs=None, f=10., phi=0.984, total_duration=4):
    """The Lorenz task in throughput mode: the graph of get_model with the two stock uniform priors
    drawn on the device and the device simulator with the six summaries fused into it; the
    Euclidean distance runs on the device.  The observed data and its summaries are computed on the
    host (the reference's default initial state and n_obs = 40).  Returns (model, DeviceModelPrior);
    pass the latter as ``device_proposal=`` to SMC."""
    y_obs = _observed(true_params, seed_obs, None, 40, f, phi, total_duration)
    simulator = partial(lorenz_device, f=f, phi=phi, total_duration=total_duration)
    m = _graph(em.new_model(), simulator, y_obs)
    dp = DeviceModelPrior(m)
    return dp.model, dp
