"""CPU test double of the Ricker entry points -- TEST INFRASTRUCTURE ONLY.

Extends tests/abi_double.py (through `abi_double.install`) with restatements of
elfi_b200_poisson_f64, elfi_b200_sim_ricker_f64, elfi_b200_count_zeros_f64 and
elfi_b200_chi_squared_f64 on host pointers.  The summaries and chi_squared are the reference's
NumPy code (elfi_b200.examples.ricker on host arrays); the simulators draw from a NumPy
RandomState instead of the device's Philox streams (same distributions, deterministic in
(seed, offset); rates the device turns into NaN give NaN here too), and the fused summaries are
those of exactly the data the unfused form writes, as on the device.
"""
import numpy as np

import abi_double as d
from elfi_b200 import ops


def _poisson(lam, rs):
    lam = np.asarray(lam, dtype=np.float64)
    bad = ~(lam >= 0.0) | (lam > ops.POISSON_LAM_MAX)
    k = rs.poisson(np.where(bad, 0.0, lam)).astype(np.float64)
    return np.where(bad, np.nan, k)


def poisson_f64(ctx, lam, n, seed, offset, out, stream):
    d._require(n >= 0, 'poisson: bad argument')
    if n:
        d._vec(out, n)[:] = _poisson(d._vec(lam, n), d._rs(seed, offset, 11))


def ricker_data(P, n_obs, stock_init, rs):
    """(Y, N): the reference's recurrences on NumPy draws."""
    B = P.shape[0]
    N = np.empty((B, n_obs))
    if P.shape[1] == 1:
        N[:, 0] = stock_init
        with np.errstate(all='ignore'):
            for t in range(1, n_obs):
                N[:, t] = N[:, t - 1] * np.exp(P[:, 0] - N[:, t - 1])
        return N.copy(), N
    Y = np.empty((B, n_obs))
    prev = np.full(B, float(stock_init))
    e = rs.randn(B, n_obs)
    with np.errstate(all='ignore'):
        for t in range(n_obs):
            prev = prev * np.exp((P[:, 0] - prev) + P[:, 1] * e[:, t])
            N[:, t] = prev
            Y[:, t] = _poisson(P[:, 2] * prev, rs)
    return Y, N


def sim_ricker_f64(ctx, P, ldP, n_params, B, n_obs, stock_init, seed, offset, Y, ldY, N, ldN, S, ldS,
                   stream):
    d._require(n_params in (1, 3), 'sim_ricker: 3 parameters or 1, got {}'.format(n_params))
    d._require(1 <= n_obs <= ops.RICKER_NOBS_MAX and ldP >= n_params, 'sim_ricker: bad shape')
    if d._addr(S):
        d._require(n_obs <= ops.RICKER_FUSED_MAX, 'sim_ricker: fused summaries need n_obs <= 128')
    if not B:
        return
    y, lat = ricker_data(d._mat(P, B, n_params, ldP).copy(), n_obs, stock_init,
                         d._rs(seed, offset, 12))
    if d._addr(Y):
        d._mat(Y, B, n_obs, ldY)[:] = y
    if d._addr(N):
        d._mat(N, B, n_obs, ldN)[:] = lat
    if d._addr(S):
        s = d._mat(S, B, 3, ldS)
        with np.errstate(invalid='ignore'):
            s[:, 0], s[:, 1] = np.mean(y, axis=1), np.var(y, axis=1)
        s[:, 2] = np.sum(y == 0, axis=1)


def count_zeros_f64(ctx, X, ldX, B, n, out, ld_out, stream):
    d._require(n >= 1 and ldX >= n, 'count_zeros: bad shape')
    if B:
        d._mat(out, B, 1, ld_out)[:, 0] = np.sum(d._mat(X, B, n, ldX) == 0, axis=1)


def chi_squared_f64(ctx, S, ldS, B, K, obs, out, stream):
    from elfi_b200.examples import ricker
    d._require(1 <= K <= 128, 'chi_squared: bad shape')
    if B:
        sim = d._mat(S, B, K, ldS)
        o = d._vec(obs, K)
        with np.errstate(divide='ignore', invalid='ignore'):
            d._vec(out, B)[:] = ricker.chi_squared(*sim.T, observed=tuple(o[:, None]))


TABLE = {'elfi_b200_' + f.__name__: f for f in (
    poisson_f64, sim_ricker_f64, count_zeros_f64, chi_squared_f64)}
