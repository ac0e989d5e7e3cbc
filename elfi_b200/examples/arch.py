"""ARCH(1) model (mirror of elfi/examples/arch.py): y_i = t1 y_{i-1} + e_i with the conditionally
heteroskedastic error e_i = xi_i sqrt(0.2 + t2 e_{i-1}^2) (Engle 1982), summarised by its mean,
variance, autocorrelations AC_1 .. AC_L and their pairwise products.

The host path (arch, E, get_model) consumes the batch's RandomState exactly as the reference does,
so it reproduces the reference's draws.  get_device_model is the same task in throughput mode: the
uniform priors drawn on the device (DeviceModelPrior), the simulator with all its summaries fused on
the device (Philox streams; statistical parity with the host path).

As in the reference, get_model's simulator is built without n_obs, so simulated series always have
100 observations while the observed one has get_model's n_obs.

sample_mean, sample_variance, autocorr and pairwise_autocorr take host arrays (the reference's
NumPy code), device tensors (ops.arch_summaries) and the lazy output of the device simulator (the
summaries computed in the simulator); all forms give the same bits."""
import logging
from functools import partial
from itertools import combinations

import numpy as np
import torch

from .. import device as dev
from .. import model as em
from .. import ops
from ..priors import DeviceModelPrior
from ..throughput import LazySimulation, batch_columns, batch_key

logger = logging.getLogger(__name__)

SIM_N_OBS = 100   # the simulator node's n_obs: get_model does not pass its own


def arch(t1, t2, n_obs=100, batch_size=1, random_state=None):
    """The ARCH(1) series (arch.py:65-105): y_0 = 0, y_i = t1 y_{i-1} + e_i for i = 1 .. n_obs;
    returns y_1 .. y_n, (batch_size, n_obs)."""
    random_state = random_state or np.random
    y = np.zeros((batch_size, n_obs + 1))
    e = E(t2, n_obs, batch_size, random_state)
    for i in range(1, n_obs + 1):
        y[:, i] = t1 * y[:, i - 1] + e[:, i]

    return y[:, 1:]


def E(t2, n_obs=100, batch_size=1, random_state=None):
    """The error process (arch.py:108-132): xi ~ N(0, 1) (batch_size, n_obs + 1) is drawn first,
    then e_0 ~ N(0, 1); e_i = xi_i sqrt(0.2 + t2 e_{i-1}^2).  Column 0 of xi is never used."""
    random_state = random_state or np.random
    xi = random_state.normal(size=(batch_size, n_obs + 1))
    e = np.zeros((batch_size, n_obs + 1))
    e[:, 0] = random_state.normal(size=batch_size)
    for i in range(1, n_obs + 1):
        e[:, i] = xi[:, i] * np.sqrt(0.2 + t2 * np.power(e[:, i - 1], 2))
    return e


def _pair_column(lag_i, lag_j, n_lags):
    return 2 + n_lags + list(combinations(range(1, n_lags + 1), 2)).index((lag_i, lag_j))


def _device_summaries(x, n_lags):
    """The (B, ops.arch_nsumm(L)) summaries of lazy simulator output or device data with at least
    n_lags lags, and L; None for host data."""
    if isinstance(x, LazySimulation):
        if n_lags <= x.n_lags:
            return x.summaries(), x.n_lags
        x = x.materialize()
    if dev.is_device_array(x):
        return ops.arch_summaries(x, n_lags=n_lags), n_lags
    return None


def sample_mean(x):
    """np.mean(x, axis=1), the summary 'MU' (arch.py:135-148)."""
    s = _device_summaries(x, 1)
    return np.mean(x, axis=1) if s is None else s[0][:, 0]


def sample_variance(x):
    """np.var(x, axis=1, ddof=1), the summary 'VAR' (arch.py:151-164)."""
    s = _device_summaries(x, 1)
    return np.var(x, axis=1, ddof=1) if s is None else s[0][:, 1]


def autocorr(x, lag=1):
    """The lag autocorrelation of the rows standardised with ddof = 1, divided by n - lag, the
    summaries 'AC_lag' (arch.py:167-187)."""
    s = _device_summaries(x, lag)
    if s is not None:
        return s[0][:, 1 + lag]
    n = x.shape[1]
    x_mu = np.mean(x, axis=1)
    x_std = np.std(x, axis=1, ddof=1)
    sc_x = ((x.T - x_mu) / x_std).T
    C = np.sum(sc_x[:, lag:] * sc_x[:, :-lag], axis=1) / (n - lag)
    return C


def pairwise_autocorr(x, lag_i=1, lag_j=1):
    """autocorr(x, lag_i) * autocorr(x, lag_j), the summaries 'PW_i_j' (arch.py:190-208)."""
    s = _device_summaries(x, max(lag_i, lag_j))
    if s is not None:
        S, n_lags = s
        if lag_i == lag_j:
            return torch.mul(S[:, 1 + lag_i], S[:, 1 + lag_i])
        return S[:, _pair_column(min(lag_i, lag_j), max(lag_i, lag_j), n_lags)]
    ac_i = autocorr(x, lag_i)
    ac_j = autocorr(x, lag_j)
    return ac_i * ac_j


def _graph(m, simulator, y_obs, n_lags):
    """Priors, simulator, summaries and distance of arch.py:36-60."""
    em.Prior('uniform', -1, 2, model=m, name='t1')
    em.Prior('uniform', 0, 1, model=m, name='t2')
    em.Simulator(simulator, m['t1'], m['t2'], observed=y_obs, name='Y')
    ss = [em.Summary(sample_mean, m['Y'], name='MU'),
          em.Summary(sample_variance, m['Y'], name='VAR')]
    for i in range(1, n_lags + 1):
        ss.append(em.Summary(autocorr, m['Y'], i, name='AC_{}'.format(i)))
    for i, j in combinations(range(1, n_lags + 1), 2):
        ss.append(em.Summary(pairwise_autocorr, m['Y'], i, j, name='PW_{}_{}'.format(i, j)))
    em.Distance('euclidean', *ss, name='d')
    return m


def _observed(n_obs, true_params, seed_obs):
    if true_params is None:
        true_params = [0.3, 0.7]
        logger.info('true_params were not given. Now using [t1, t2] = {}.'.format(true_params))
    return arch(*true_params, n_obs=n_obs, random_state=np.random.RandomState(seed_obs))


def get_model(n_obs=100, true_params=None, seed_obs=None, n_lags=5):
    """The ARCH(1) inference task of arch.py:13-62: uniform priors t1 on [-1, 1] and t2 on [0, 1],
    the simulator 'Y', the summaries MU, VAR, AC_1 .. AC_L and PW_i_j, and the Euclidean distance
    'd'.  The observed series has n_obs observations, simulated ones always 100."""
    y_obs = _observed(n_obs, true_params, seed_obs)
    return _graph(em.new_model(), arch, y_obs, n_lags)


# ---------------------------------------------------------------------------- throughput mode
def arch_device(t1, t2, n_lags=5, batch_size=1, random_state=None):
    """Device twin of arch (100 observations, as the simulator node of get_model draws); returns a
    LazySimulation of shape (batch_size, 100) whose summaries [MU, VAR, AC_1 .. AC_L, PW] are
    computed in the simulator kernel."""
    P = torch.stack(batch_columns((t1, t2), batch_size), dim=1)
    key = batch_key(random_state)
    lazy = LazySimulation(
        (int(P.shape[0]), SIM_N_OBS),
        lambda kind: ops.sim_arch(P, SIM_N_OBS, n_lags, seed=key)[1],
        lambda: ops.sim_arch(P, SIM_N_OBS, n_lags, seed=key, want_data=True,
                             want_summaries=False)[0])
    lazy.n_lags = n_lags
    return lazy


def get_device_model(n_obs=100, true_params=None, seed_obs=None, n_lags=5):
    """The ARCH(1) task in throughput mode: the graph of get_model with the uniform priors drawn on
    the device and the device simulator with all its summaries fused into it.  The observed data
    and its summaries are computed on the host.  Returns (model, DeviceModelPrior); pass the latter
    as ``device_proposal=`` to SMC."""
    ops._arch_shape(SIM_N_OBS, n_lags, 'the device ARCH simulator and its summaries')
    y_obs = _observed(n_obs, true_params, seed_obs)
    m = _graph(em.new_model(), partial(arch_device, n_lags=n_lags), y_obs, n_lags)
    dp = DeviceModelPrior(m)
    return dp.model, dp
