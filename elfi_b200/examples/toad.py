"""Toad movement model (mirror of elfi/examples/toad.py; Marchand et al. 2017): n_toads Fowler's
toads over n_days days.  Each day a toad either returns to the refuge of a uniformly chosen earlier
day (probability p0) or takes a symmetric alpha-stable step of scale gamma from yesterday's
position.  Four summaries compare the displacements over 1, 2, 4 and 8 days.

The host path (toad, compute_summaries, get_model) consumes the batch's RandomState exactly as the
reference does, so it reproduces the reference's draws.  The reference assigns
``scipy.stats.levy_stable.random_state``, a SciPy global; here the RandomState is passed to ``rvs``
instead, which gives the same draws.  get_device_model is the same task in throughput mode: the
stock priors drawn on the device (DeviceModelPrior), the simulator with its summaries fused on the
device (Philox streams; statistical parity with the host path).

compute_summaries takes host arrays (the reference's NumPy code), device tensors
(ops.toad_summaries) and the lazy output of the device simulator (the summaries computed in the
simulator); all forms give the same values."""
import warnings
from functools import partial

import numpy as np
import scipy.stats as ss
import torch

from .. import device as dev
from .. import model as em
from .. import ops
from ..priors import DeviceModelPrior
from ..throughput import LazySimulation, batch_columns, batch_key

P_DEFAULT = np.linspace(0, 1, 11)
P_DEFAULT.setflags(write=False)
THD_DEFAULT = 10
LAGS = (1, 2, 4, 8)   # the summary nodes S1, S2, S4, S8


def toad(alpha, gamma, p0, n_toads=66, n_days=63, batch_size=1, random_state=None):
    """The toad movement simulator (toad.py:16-70): (n_days, n_toads, batch_size), batch last.

    Day 0 is 0 for every toad.  Day i draws, in this order, the return uniforms (n_toads, B), the
    levy_stable(alpha, beta=0, scale=gamma) steps (a uniform angle, then a standard exponential)
    and the refuge days choice(i).  A returning toad (uniform < p0) takes its position of the
    refuge day, the others step from day i - 1."""
    X = np.zeros((n_days, n_toads, batch_size))
    random_state = random_state or np.random

    for i in range(1, n_days):
        ret = random_state.uniform(0, 1, (n_toads, batch_size)) < np.squeeze(p0)
        non_ret = np.invert(ret)

        delta_x = ss.levy_stable.rvs(alpha, beta=0, scale=gamma, size=(n_toads, batch_size),
                                     random_state=random_state)
        X[i, non_ret] = X[i - 1, non_ret] + delta_x[non_ret]

        ind_refuge = random_state.choice(i, size=(n_toads, batch_size))
        X[i, ret] = X[ind_refuge[ret], ret]

    return X


def obs_mat_to_deltax(X, lag):
    """The displacements over lag days (toad.py:116-132): X[lag:] - X[:-lag] as
    (n_toads * (n_days - lag), batch_size)."""
    batch_size = np.atleast_3d(X).shape[-1]
    return (X[lag:] - X[:-lag]).reshape(-1, batch_size)


def _host_summaries(X, lag, p, thd):
    abs_disp = np.abs(obs_mat_to_deltax(X, lag))
    # a displacement below thd is a return to a refuge
    ret = abs_disp < thd
    num_ret = np.sum(ret, axis=0)
    # the other displacements, without the returns and the NaNs
    abs_disp[ret] = np.nan
    with warnings.catch_warnings():
        warnings.filterwarnings('ignore', r'All-NaN slice encountered')
        abs_noret_median = np.nanmedian(abs_disp, axis=0)
        abs_noret_quantiles = np.nanquantile(abs_disp, p, axis=0)
    diff = np.diff(abs_noret_quantiles, axis=0)
    # zero gaps are floored at exp(-20) before the log
    logdiff = np.log(np.maximum(diff, np.exp(-20)))
    ssx = np.vstack((num_ret, abs_noret_median, logdiff))
    # NaN where every toad returned
    ssx = np.nan_to_num(ssx, nan=np.inf)
    return np.transpose(ssx)


def _is_fused_set(lag, p, thd):
    return (lag in LAGS and thd == THD_DEFAULT and np.shape(p) == P_DEFAULT.shape
            and np.array_equal(np.asarray(p, dtype=np.float64), P_DEFAULT))


def compute_summaries(X, lag, p=P_DEFAULT, thd=THD_DEFAULT):
    """The summaries of the displacements over lag days (toad.py:73-113), (batch_size, len(p) + 1):
    the number of returns (|displacement| < thd), the median of the other absolute displacements,
    and the logs of the gaps between their p quantiles (floored at exp(-20)); NaN becomes inf,
    +-inf the largest finite double.

    Lazy device output gives its columns of the fused summaries when (lag, p, thd) is one of the
    fused sets (lag in 1, 2, 4, 8 with the default p and thd), otherwise the summaries of its
    data.  Device data goes to ops.toad_summaries, host data to NumPy."""
    if isinstance(X, LazySimulation):
        lags = _fused_lags(X.shape[0])
        if _is_fused_set(lag, p, thd) and lag in lags:
            w = len(P_DEFAULT) + 1
            j = lags.index(lag)
            return X.summaries()[:, j * w:(j + 1) * w]
        X = X.materialize()
    if dev.is_device_array(X):
        return ops.toad_summaries(X, lag, p, thd)
    return _host_summaries(X, lag, p, thd)


def _graph(m, simulator, y_obs):
    """Priors, simulator, summaries and discrepancy of toad.py:154-167."""
    em.Prior('uniform', 1, 1, model=m, name='alpha')
    em.Prior('uniform', 0, 100, model=m, name='gamma')
    em.Prior('uniform', 0, 0.9, model=m, name='p0')
    em.Simulator(simulator, m['alpha'], m['gamma'], m['p0'], observed=y_obs, name='toad')
    sumstats = [em.Summary(partial(compute_summaries, lag=lag), m['toad'], name='S{}'.format(lag))
                for lag in LAGS]
    em.Distance('euclidean', *sumstats, name='d')
    return m


def _observed(true_params, seed_obs):
    if true_params is None:
        true_params = [1.7, 35.0, 0.6]
    return toad(*true_params, random_state=np.random.RandomState(seed_obs))


def get_model(true_params=None, seed_obs=None):
    """The toad inference task of toad.py:135-172: uniform priors on alpha (1, 2), gamma (0, 100)
    and p0 (0, 0.9), the simulator 'toad', the summaries S1, S2, S4, S8 and the Euclidean distance
    'd'."""
    return _graph(em.new_model(), toad, _observed(true_params, seed_obs))


# ---------------------------------------------------------------------------- throughput mode
def _fused_lags(n_days):
    return tuple(lag for lag in LAGS if lag < n_days)


def toad_device(alpha, gamma, p0, n_toads=66, n_days=63, batch_size=1, random_state=None):
    """Device twin of toad; returns a LazySimulation of shape (n_days, n_toads, batch_size) whose
    summaries for lags 1, 2, 4, 8 (default p and thd) are computed in the simulator kernel.
    materialize() gives the data as a (n_days, n_toads, batch_size) view of the batch-major
    kernel output, indexed like the reference's array."""
    P = torch.stack(batch_columns((alpha, gamma, p0), batch_size), dim=1)
    key = batch_key(random_state)
    lags = _fused_lags(n_days)
    return LazySimulation(
        (int(n_days), int(n_toads), int(P.shape[0])),
        lambda kind: ops.sim_toad(P, n_toads, n_days, seed=key, lags=lags, p=P_DEFAULT,
                                  thd=THD_DEFAULT)[1],
        lambda: ops.sim_toad(P, n_toads, n_days, seed=key, want_data=True,
                             lags=None)[0].permute(1, 2, 0))


def get_device_model(true_params=None, seed_obs=None):
    """The toad task in throughput mode: the graph of get_model with the three stock uniform priors
    drawn on the device and the device simulator with the four summaries fused into it; the
    Euclidean distance runs on the device.  The observed data and its summaries are computed on the
    host.  Returns (model, DeviceModelPrior); pass the latter as ``device_proposal=`` to SMC."""
    m = _graph(em.new_model(), toad_device, _observed(true_params, seed_obs))
    dp = DeviceModelPrior(m)
    return dp.model, dp
