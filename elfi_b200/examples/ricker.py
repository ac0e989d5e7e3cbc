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
all forms give the same bits.

ss_wood is the set of 13 statistics Wood (2010) introduced synthetic likelihood with; the reference
points to it but ships only Mean, Var and #0.  get_model(summary='wood') and
get_device_model(summary='wood') build the task with it, for BSL."""
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


# ---------------------------------------------------------------------------- Wood (2010)
WOOD_NOBS_MIN = 7
_WOOD_DESIGNS = {}   # id(observed series) -> [the series, its values, host design, device design]


def wood_design(obs_series):
    """The (3, n - 1) pseudo-inverse of [o, o^2, o^3], o = np.sort(np.diff(obs_series)): the map from
    the sorted differences of a simulated series to their cubic regression on o."""
    o = np.sort(np.diff(np.asarray(obs_series, dtype=np.float64).reshape(-1)))
    return np.ascontiguousarray(np.linalg.pinv(np.column_stack([o, o ** 2, o ** 3])))


def _wood_design(obs_series, n, on_device):
    """wood_design of an observed series of n values, made once per series (and copied to the
    device once)."""
    hit = _WOOD_DESIGNS.get(id(obs_series))
    if hit is None or hit[0] is not obs_series:
        obs = np.asarray(obs_series, dtype=np.float64)
        if obs.ndim > 2 or (obs.ndim == 2 and obs.shape[0] != 1):
            raise ValueError('the observed series must be one row, got shape {}'.format(obs.shape))
        if len(_WOOD_DESIGNS) > 64:
            _WOOD_DESIGNS.clear()
        hit = [obs_series, obs.reshape(-1), None, None]
        _WOOD_DESIGNS[id(obs_series)] = hit
    if hit[1].size != n:
        raise ValueError('the observed series has {} values, the simulated series {}'.format(
            hit[1].size, n))
    if hit[2] is None:
        hit[2] = wood_design(hit[1])
    if on_device and hit[3] is None:
        hit[3] = dev.to_device(hit[2])
    return hit[3] if on_device else hit[2]


def wood_statistics(y, design):
    """ss_wood of host data y (B, n) with the cubic design of its observed series precomputed
    (wood_design): the vectorised NumPy definition of the 13 statistics, (B, 13)."""
    y = np.ascontiguousarray(np.atleast_2d(y), dtype=np.float64)
    B, n = y.shape
    if n < WOOD_NOBS_MIN:
        raise ValueError("Wood's statistics take n_obs >= {}, got {}".format(WOOD_NOBS_MIN, n))
    out = np.empty((B, 13))
    with np.errstate(all='ignore'):
        m = np.mean(y, axis=1)
        out[:, 0] = m
        out[:, 1] = np.sum(y == 0, axis=1)
        yc = y - m[:, None]
        for k in range(6):
            out[:, 2 + k] = np.sum(yc[:, :n - k] * yc[:, k:], axis=1) / n
        e = np.sort(np.diff(y, axis=1), axis=1)
        out[:, 8:11] = e @ np.asarray(design).T
        x, w = y[:, :-1], y[:, 1:] ** 0.3
        u, v = x ** 0.3, x ** 0.6
        suu, suv, svv = np.sum(u * u, axis=1), np.sum(u * v, axis=1), np.sum(v * v, axis=1)
        suw, svw = np.sum(u * w, axis=1), np.sum(v * w, axis=1)
        det = suu * svv - suv * suv
        a1 = (svv * suw - suv * svw) / det
        a2 = (suu * svw - suv * suw) / det
        # the rank rule: N = the distinct nonzero values of y[:-1]
        nz = x != 0
        some = nz.any(axis=1)
        k = x[np.arange(B), np.argmax(nz, axis=1)]
        one = some & ~np.any(nz & (x != k[:, None]), axis=1)
        at_k = x == k[:, None]
        s = np.sum(np.where(at_k, w, 0.0), axis=1) / np.sum(at_k, axis=1)
        den = k ** 0.6 + k ** 1.2
        out[:, 11] = np.where(one, s * k ** 0.3 / den, np.where(some, a1, 0.0))
        out[:, 12] = np.where(one, s * k ** 0.6 / den, np.where(some, a2, 0.0))
    out[~np.isfinite(y).all(axis=1)] = np.nan
    return out


def ss_wood(y, obs_series):
    """The 13 summary statistics of Wood (2010, Nature 466:1102) for a Ricker series y (B, n) and
    the observed series of the same length n >= 7, in this project's reading of the paper (which
    leaves divisors, lags, intercepts and degenerate cases open).  Columns:

    * 0: the mean; 1: the number of zeros;
    * 2..7: the autocovariances sum_t (y_t - m)(y_{t+k} - m) / n at lags k = 0..5 (lag 0 is np.var);
    * 8..10: the cubic regression, without intercept, of the sorted differences
      np.sort(np.diff(y)) on the sorted observed differences o: their product with the
      pseudo-inverse of [o, o^2, o^3] (wood_design);
    * 11..12: the autoregression y_{t+1}^0.3 = a1 y_t^0.3 + a2 y_t^0.6, without intercept, by
      minimum-norm least squares.  With N the distinct nonzero values of y[:-1]: N empty gives
      (0, 0); N = {k} (proportional columns) gives s (k^0.3, k^0.6) / (k^0.6 + k^1.2), s the mean
      of y_{t+1}^0.3 over the t with y_t = k; otherwise the normal equations.

    A row with a non-finite value gives 13 NaN.  Host arrays take the NumPy definition
    (wood_statistics), device tensors and the lazy output of the device simulator the kernel
    (ops.wood_summaries, n <= ops.RICKER_WOOD_NOBS_MAX), which matches it to the accuracy stated
    in include/elfi_b200.h.  The design is computed once per observed series."""
    if isinstance(y, LazySimulation):
        y = y.materialize()
    on_device = dev.is_device_array(y)
    if not on_device:
        y = np.atleast_2d(y)
    n = int(y.shape[-1])
    if n < WOOD_NOBS_MIN:
        raise ValueError("Wood's statistics take n_obs >= {}, got {}".format(WOOD_NOBS_MIN, n))
    design = _wood_design(obs_series, n, on_device)
    return ops.wood_summaries(y, design) if on_device else wood_statistics(y, design)


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


SUMMARIES = ('chi_squared', 'wood')


def _check_summary(summary, stochastic, n_obs):
    if summary not in SUMMARIES:
        raise ValueError("summary must be 'chi_squared' or 'wood', got {!r}".format(summary))
    if summary == 'wood':
        if not stochastic:
            raise ValueError("summary='wood' needs the stochastic model")
        if n_obs < WOOD_NOBS_MIN:
            raise ValueError("Wood's statistics take n_obs >= {}, got {}".format(WOOD_NOBS_MIN,
                                                                                  n_obs))


def _graph(m, simulator, y_obs, stochastic, summary='chi_squared'):
    """Priors, simulator, summaries and discrepancy of ricker.py:128-142; with summary='wood' the
    summary node 'Wood' (ss_wood, 13 columns) and no discrepancy (for BSL)."""
    if stochastic:
        em.Prior(ss.expon, np.e, 2, model=m, name='t1')
        em.Prior(ss.truncnorm, 0, 5, model=m, name='t2')
        em.Prior(ss.uniform, 0, 100, model=m, name='t3')
        em.Simulator(simulator, m['t1'], m['t2'], m['t3'], observed=y_obs, name='Ricker')
        if summary == 'wood':
            em.Summary(partial(ss_wood, obs_series=y_obs), m['Ricker'], name='Wood')
            return m
        sumstats = [em.Summary(ss_mean, m['Ricker'], name='Mean'),
                    em.Summary(ss_var, m['Ricker'], name='Var'),
                    em.Summary(num_zeros, m['Ricker'], name='#0')]
        em.Discrepancy(chi_squared, *sumstats, name='d')
    else:
        em.Prior(ss.expon, np.e, model=m, name='t1')
        em.Simulator(simulator, m['t1'], observed=y_obs, name='Ricker')
        em.Distance('euclidean', em.Summary(ss_mean, m['Ricker'], name='Mean'), name='d')
    return m


def get_model(n_obs=50, true_params=None, seed_obs=None, stochastic=True, summary='chi_squared'):
    """The Ricker inference task of ricker.py:88-144: the stochastic model with Mean, Var, #0 and
    chi_squared, or (stochastic=False) the deterministic map with Mean and the Euclidean
    distance.  summary='wood' (stochastic model, n_obs >= 7) replaces the summaries and the
    discrepancy by one summary node 'Wood', Wood's 13 statistics (ss_wood), for
    BSL(m, n_sim_round, ['Wood']).  Their variances span ~16 orders of magnitude, beyond the
    synthetic likelihood's pivot cut, so give BSL a common scale, e.g.
    bsl.standard_likelihood(whitening=np.diag(1 / sd)) with sd their standard deviations in a pilot
    run at a plausible parameter."""
    _check_summary(summary, stochastic, n_obs)
    y_obs = _observed(n_obs, true_params, seed_obs, stochastic)
    simulator = partial(stochastic_ricker if stochastic else ricker, n_obs=n_obs)
    return _graph(em.new_model(), simulator, y_obs, stochastic, summary)


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


def get_device_model(n_obs=50, true_params=None, seed_obs=None, stochastic=True,
                     summary='chi_squared'):
    """The Ricker task in throughput mode: the graph of get_model with the stock priors drawn on the
    device, the device simulator with Mean, Var and #0 fused into it, and chi_squared (or the
    Euclidean distance) on the device.  summary='wood' gives the summary node 'Wood' instead, Wood's
    13 statistics computed by the device kernel on the simulated counts (7 <= n_obs <=
    ops.RICKER_WOOD_NOBS_MAX), for BSL.  The observed data and its summaries are computed on the
    host.  Returns (model, DeviceModelPrior); pass the latter as ``device_proposal=`` to SMC or
    BSL."""
    if not 1 <= n_obs <= ops.RICKER_NOBS_MAX:
        raise ValueError('the device Ricker simulator takes 1 <= n_obs <= {}, got {}'.format(
            ops.RICKER_NOBS_MAX, n_obs))
    _check_summary(summary, stochastic, n_obs)
    if summary == 'wood' and n_obs > ops.RICKER_WOOD_NOBS_MAX:
        raise ValueError("Wood's statistics on the device take n_obs <= {}, got {}".format(
            ops.RICKER_WOOD_NOBS_MAX, n_obs))
    y_obs = _observed(n_obs, true_params, seed_obs, stochastic)
    simulator = partial(ricker_device, n_obs=n_obs, stochastic=stochastic)
    m = _graph(em.new_model(), simulator, y_obs, stochastic, summary)
    dp = DeviceModelPrior(m)
    return dp.model, dp
