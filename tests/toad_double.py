"""CPU test double of the toad entry points -- TEST INFRASTRUCTURE ONLY.

Extends tests/abi_double.py (through `abi_double.install`) with restatements of
elfi_b200_sim_toad_f64 and elfi_b200_toad_summaries_f64 on host pointers.  The summaries are the
reference's NumPy code (elfi_b200.examples.toad on host arrays); the simulator is the reference's
toad() on a NumPy RandomState instead of the device's Philox streams (same distribution,
deterministic in (seed, offset)), with NaN rows where the device gives them, and the fused summaries
are those of exactly the data the unfused form writes, as on the device.
"""
import numpy as np

import abi_double as d
from elfi_b200 import ops


def toad_data(P, n_toads, n_days, rs):
    from elfi_b200.examples import toad
    alpha, gamma, p0 = P[:, 0].copy(), P[:, 1].copy(), P[:, 2].copy()
    bad = ~((alpha > 0) & (alpha <= 2) & (gamma >= 0))
    alpha[bad], gamma[bad] = 1.5, 1.0
    with np.errstate(all='ignore'):
        X = toad.toad(alpha, gamma, p0, n_toads=n_toads, n_days=n_days, batch_size=len(P),
                      random_state=rs)
    X[:, :, bad] = np.nan
    return np.ascontiguousarray(X.transpose(2, 0, 1))      # (B, n_days, n_toads)


def _summaries(x, lag, p, thd):
    from elfi_b200.examples import toad
    with np.errstate(all='ignore'):
        return toad.compute_summaries(x, lag, p=p, thd=thd)


def sim_toad_f64(ctx, P, ldP, B, n_toads, n_days, seed, offset, X, n_lags, lags, n_p, p, thd, S,
                 ldS, stream):
    d._require(ldP >= 3 and n_toads >= 1 and n_days >= 1 and
               n_toads * n_days <= ops.TOAD_CELLS_MAX, 'sim_toad: bad shape')
    if d._addr(S):
        lg = d._vec(lags, n_lags, dtype=np.int64)
        d._require(1 <= n_lags <= ops.TOAD_LAGS_MAX and 1 <= n_p <= ops.TOAD_NP_MAX and
                   ldS >= n_lags * (n_p + 1) and n_toads * (n_days - 1) <= ops.TOAD_DISP_MAX and
                   np.all((lg >= 1) & (lg < n_days)), 'sim_toad: bad summaries')
    if not B or not (d._addr(X) or d._addr(S)):
        return
    x = toad_data(d._mat(P, B, 3, ldP).copy(), n_toads, n_days, d._rs(seed, offset, 17))
    if d._addr(X):
        d._mat(X, B, n_days * n_toads)[:] = x.reshape(B, -1)
    if d._addr(S):
        pv = d._vec(p, n_p).copy()
        w = n_p + 1
        out = d._mat(S, B, n_lags * w, ldS)
        xr = x.transpose(1, 2, 0)
        for j, lag in enumerate(lg):
            out[:, j * w:(j + 1) * w] = _summaries(xr, int(lag), pv, thd)


def toad_summaries_f64(ctx, X, ld_day, ld_toad, ld_row, n_days, n_toads, B, lag, n_p, p, thd, S,
                       ldS, stream):
    d._require(1 <= lag < n_days and n_toads * (n_days - lag) <= ops.TOAD_DISP_MAX and
               1 <= n_p <= ops.TOAD_NP_MAX and ldS >= n_p + 1, 'toad_summaries: bad shape')
    if not B:
        return
    span = (n_days - 1) * ld_day + (n_toads - 1) * ld_toad + (B - 1) * ld_row + 1
    x = np.lib.stride_tricks.as_strided(d._vec(X, span), (n_days, n_toads, B),
                                        (8 * ld_day, 8 * ld_toad, 8 * ld_row))
    d._mat(S, B, n_p + 1, ldS)[:] = _summaries(np.array(x), lag, d._vec(p, n_p).copy(), thd)


TABLE = {'elfi_b200_' + f.__name__: f for f in (sim_toad_f64, toad_summaries_f64)}
