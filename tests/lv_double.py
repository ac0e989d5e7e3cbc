"""CPU test double of the Lotka-Volterra entry points -- TEST INFRASTRUCTURE ONLY.

Extends tests/abi_double.py (through `abi_double.install`) with restatements of
elfi_b200_sim_lotka_volterra_f64 and elfi_b200_lv_summaries_f64 on host pointers.  The summaries
are the reference's NumPy code (elfi_b200.examples.lotka_volterra on host arrays); the simulator is
the reference's lotka_volterra() on a NumPy RandomState instead of the device's Philox streams (same
distribution, deterministic in (seed, offset)), with NaN rows where the device gives them: rejected
parameters, and rows that need more than max_events events (n_events = max_events).
"""
import numpy as np

import abi_double as d
from elfi_b200 import ops


def lv_data(P, n_obs, time_end, max_events, rs):
    from elfi_b200.examples import lotka_volterra as lv
    P = P.copy()
    with np.errstate(invalid='ignore'):
        X0, Y0 = np.floor(P[:, 3]), np.floor(P[:, 4])
        bad = ~((P[:, :3] >= 0).all(axis=1) & (P[:, 5] >= 0) & (X0 >= 0) & (X0 < 2 ** 31)
                & (Y0 >= 0) & (Y0 < 2 ** 31))
    P[bad] = [1.0, 0.005, 0.6, 50, 100, 0.0]
    with np.errstate(all='ignore'):
        obs, _, _, times = lv.lotka_volterra(*P.T, n_obs=n_obs, time_end=time_end,
                                             batch_size=len(P), random_state=rs, return_full=True)
    n_events = np.argmax(times >= time_end, axis=1).astype(np.int64)
    obs = obs.astype(np.float64)
    capped = n_events > max_events
    obs[bad | capped] = np.nan
    n_events[bad] = 0
    n_events[capped] = max_events
    return obs, n_events


def sim_lotka_volterra_f64(ctx, P, ldP, B, t_out, n_obs, time_end, max_events, seed, offset, X,
                           n_events, stream):
    d._require(ldP >= 6 and 1 <= n_obs <= ops.LV_NOBS_MAX and 0 < time_end < np.inf and
               1 <= max_events <= ops.LV_MAX_EVENTS_LIMIT, 'sim_lotka_volterra: bad shape')
    if not B:
        return
    d._require(np.array_equal(d._vec(t_out, n_obs), np.linspace(0, time_end, n_obs)),
               'sim_lotka_volterra: t_out is not np.linspace(0, time_end, n_obs)')
    obs, n = lv_data(d._mat(P, B, 6, ldP).copy(), n_obs, time_end, max_events,
                     d._rs(seed, offset, 23))
    d._mat(X, B, 2 * n_obs)[:] = obs.reshape(B, -1)
    d._vec(n_events, B, np.int64)[:] = n


def lv_summaries_f64(ctx, X, ld_row, ld_obs, ld_species, B, n_obs, S, ldS, stream):
    from elfi_b200.examples import lotka_volterra as lv
    d._require(ops.LV_SUMM_NOBS_MIN <= n_obs <= ops.LV_SUMM_NOBS_MAX and ldS >= ops.LV_NSUMM,
               'lv_summaries: bad shape')
    if not B:
        return
    span = (B - 1) * ld_row + (n_obs - 1) * ld_obs + ld_species + 1
    x = np.array(np.lib.stride_tricks.as_strided(d._vec(X, span), (B, n_obs, 2),
                                                 (8 * ld_row, 8 * ld_obs, 8 * ld_species)))
    with np.errstate(all='ignore'):
        cols = [lv.stock_mean(x, 0), lv.stock_mean(x, 1), lv.stock_log_variance(x, 0),
                lv.stock_log_variance(x, 1), lv.stock_autocorr(x, 0, 1), lv.stock_autocorr(x, 1, 1),
                lv.stock_autocorr(x, 0, 2), lv.stock_autocorr(x, 1, 2), lv.stock_crosscorr(x)]
    d._mat(S, B, ops.LV_NSUMM, ldS)[:] = np.column_stack(cols)


TABLE = {'elfi_b200_' + f.__name__: f for f in (sim_lotka_volterra_f64, lv_summaries_f64)}
