"""Ricker population model (mirror of elfi/examples/ricker.py): a latent stock
N_t = N_{t-1} exp(r - N_{t-1} + sigma e_t) observed as Poisson(phi N_t) counts (Ricker 1954; Wood
2010), or the deterministic map N_t = N_{t-1} exp(r - N_{t-1}).

The host path (ricker, stochastic_ricker, get_model) consumes the batch's RandomState exactly as
the reference does, so it reproduces the reference's draws.  get_device_model is the same task in
throughput mode: the stock priors drawn on the device (DeviceModelPrior), the simulator with its
summaries fused on the device (Philox streams; statistical parity with the host path).

ss_mean, ss_var and num_zeros (the reference's Summary(partial(np.mean, axis=1)), np.var and
num_zeros) and chi_squared take host arrays (the reference's NumPy code), device tensors (the
kernels) and the lazy output of the device simulator (the summaries computed in the simulator);
all forms give the same bits."""
from functools import partial

import numpy as np
import scipy.stats as ss
import torch

from .. import device as dev
from .. import model as em
from .. import ops
from ..priors import DeviceModelPrior
from ..throughput import LazySimulation, batch_columns, batch_key


def ricker(log_rate, stock_init=1., n_obs=50, batch_size=1, random_state=None):
    """The deterministic Ricker map (ricker.py:11-40): column 0 is stock_init, then
    stock_t = stock_{t-1} exp(log_rate - stock_{t-1}); (batch_size, n_obs)."""
    random_state = random_state or np.random

    stock = np.empty((batch_size, n_obs))
    stock[:, 0] = stock_init

    for ii in range(1, n_obs):
        stock[:, ii] = stock[:, ii - 1] * np.exp(log_rate - stock[:, ii - 1])

    return stock


def stochastic_ricker(log_rate, std, scale, stock_init=1., n_obs=50, batch_size=1,
                      random_state=None):
    """The stochastic Ricker model (ricker.py:43-85): n_obs new Poisson(scale * stock) counts,
    (batch_size, n_obs)."""
    random_state = random_state or np.random

    stock_obs = np.empty((batch_size, n_obs))
    stock_prev = stock_init

    for ii in range(n_obs):
        stock = stock_prev * np.exp(log_rate - stock_prev + std * random_state.randn(batch_size))
        stock_prev = stock

        # the observed stock is Poisson distributed
        stock_obs[:, ii] = random_state.poisson(scale * stock, batch_size)

    return stock_obs


def _summary(y, col):
    """Column col of [mean, var, #0] for lazy simulator output or device data; None for host data."""
    if isinstance(y, LazySimulation):
        return y.summaries()[:, col]
    if dev.is_device_array(y):
        return ops.meanvar(y)[:, col] if col < 2 else ops.count_zeros(y)
    return None


def ss_mean(y):
    """np.mean(y, axis=1), the summary 'Mean' (ricker.py:133)."""
    s = _summary(y, 0)
    return np.mean(y, axis=1) if s is None else s


def ss_var(y):
    """np.var(y, axis=1), the summary 'Var' (ricker.py:134)."""
    s = _summary(y, 1)
    return np.var(y, axis=1) if s is None else s


def num_zeros(x):
    """The number of zero observations per row (ricker.py:164-167); float64 on the device."""
    s = _summary(x, 2)
    if s is not None:
        return s
    n = np.sum(x == 0, axis=1)
    return n


def chi_squared(*simulated, observed):
    """Chi-squared goodness of fit (ricker.py:147-161); device summaries give a device (B,)
    result."""
    if any(dev.is_device_array(s) for s in simulated):
        return ops.chi_squared(em._stack_summaries(simulated), em._stack_observed(observed))
    simulated = np.column_stack(simulated)
    observed = np.column_stack(observed)
    d = np.sum((simulated - observed)**2. / observed, axis=1)
    return d


def _observed(n_obs, true_params, seed_obs, stochastic):
    if stochastic:
        simulator = partial(stochastic_ricker, n_obs=n_obs)
        if true_params is None:
            true_params = [3.8, 0.3, 10.]
    else:
        simulator = partial(ricker, n_obs=n_obs)
        if true_params is None:
            true_params = [3.8]
    return simulator(*true_params, n_obs=n_obs, random_state=np.random.RandomState(seed_obs))


def _graph(m, simulator, y_obs, stochastic):
    """Priors, simulator, summaries and discrepancy of ricker.py:128-142."""
    if stochastic:
        em.Prior(ss.expon, np.e, 2, model=m, name='t1')
        em.Prior(ss.truncnorm, 0, 5, model=m, name='t2')
        em.Prior(ss.uniform, 0, 100, model=m, name='t3')
        em.Simulator(simulator, m['t1'], m['t2'], m['t3'], observed=y_obs, name='Ricker')
        sumstats = [em.Summary(ss_mean, m['Ricker'], name='Mean'),
                    em.Summary(ss_var, m['Ricker'], name='Var'),
                    em.Summary(num_zeros, m['Ricker'], name='#0')]
        em.Discrepancy(chi_squared, *sumstats, name='d')
    else:
        em.Prior(ss.expon, np.e, model=m, name='t1')
        em.Simulator(simulator, m['t1'], observed=y_obs, name='Ricker')
        em.Distance('euclidean', em.Summary(ss_mean, m['Ricker'], name='Mean'), name='d')
    return m


def get_model(n_obs=50, true_params=None, seed_obs=None, stochastic=True):
    """The Ricker inference task of ricker.py:88-144: the stochastic model with Mean, Var, #0 and
    chi_squared, or (stochastic=False) the deterministic map with Mean and the Euclidean
    distance."""
    y_obs = _observed(n_obs, true_params, seed_obs, stochastic)
    simulator = partial(stochastic_ricker if stochastic else ricker, n_obs=n_obs)
    return _graph(em.new_model(), simulator, y_obs, stochastic)


# ---------------------------------------------------------------------------- throughput mode
def ricker_device(*params, n_obs=50, stochastic=True, batch_size=1, random_state=None):
    """Device twin of stochastic_ricker (params log_rate, std, scale) or, with stochastic=False,
    of ricker (log_rate); returns a LazySimulation of shape (batch_size, n_obs) whose summaries
    are [mean, var, #0], computed in the simulator kernel for n_obs <= ops.RICKER_FUSED_MAX."""
    P = torch.stack(batch_columns(params, batch_size), dim=1)
    key = batch_key(random_state)
    return LazySimulation(
        (int(P.shape[0]), n_obs),
        lambda kind: ops.sim_ricker(P, n_obs, seed=key, stochastic=stochastic)[2],
        lambda: ops.sim_ricker(P, n_obs, seed=key, stochastic=stochastic, want_data=True,
                               want_summaries=False)[0])


def get_device_model(n_obs=50, true_params=None, seed_obs=None, stochastic=True):
    """The Ricker task in throughput mode: the graph of get_model with the stock priors drawn on the
    device, the device simulator with Mean, Var and #0 fused into it, and chi_squared (or the
    Euclidean distance) on the device.  The observed data and its summaries are computed on the
    host.  Returns (model, DeviceModelPrior); pass the latter as ``device_proposal=`` to SMC."""
    if not 1 <= n_obs <= ops.RICKER_NOBS_MAX:
        raise ValueError('the device Ricker simulator takes 1 <= n_obs <= {}, got {}'.format(
            ops.RICKER_NOBS_MAX, n_obs))
    y_obs = _observed(n_obs, true_params, seed_obs, stochastic)
    simulator = partial(ricker_device, n_obs=n_obs, stochastic=stochastic)
    m = _graph(em.new_model(), simulator, y_obs, stochastic)
    dp = DeviceModelPrior(m)
    return dp.model, dp
