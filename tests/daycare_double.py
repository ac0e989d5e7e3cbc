"""CPU test double of the day care entry points -- TEST INFRASTRUCTURE ONLY.

Extends tests/abi_double.py (through `abi_double.install`) with restatements of
elfi_b200_sim_daycare_f64, elfi_b200_daycare_summaries_f64 and elfi_b200_daycare_distance_f64 on
host pointers.  The summaries and the distance are the reference's NumPy code
(elfi_b200.examples.daycare on host arrays); the simulator is the reference's daycare() run one row
at a time (batch_size=1, the device's law) on a NumPy RandomState instead of the device's Philox
streams (same distribution, deterministic in (seed, offset)), with K the transitions of the row and
NaN summaries, zero data and K = -1 for the rows the device refuses (daycare_replay.row_ok).
"""
import numpy as np

import abi_double as d
from elfi_b200 import ops


def _summaries(x):
    from elfi_b200.examples import daycare as dc
    with np.errstate(all='ignore'):
        return np.concatenate([dc.ss_shannon(x), dc.ss_strains(x), dc.ss_prevalence(x),
                               dc.ss_prevalence_multi(x)], axis=1)


def sim_daycare_f64(ctx, P, ldP, B, n_dcc, n_ind, n_strains, freq, n_obs, time_end, seed, offset,
                    S, ldS, X, K, stream):
    from elfi_b200.examples import daycare as dc
    d._require(ldP >= 3 and 1 <= n_dcc <= ops.DC_DCC_MAX and 2 <= n_ind <= ops.DC_IND_MAX and
               1 <= n_strains <= ops.DC_STRAINS_MAX and 1 <= n_obs <= n_ind and
               0 < time_end < np.inf, 'sim_daycare: bad shape')
    if not B:
        return
    P = d._mat(P, B, 3, ldP)
    f = d._vec(freq, n_strains).copy()
    rs = d._rs(seed, offset, 29)
    data = np.zeros((B, n_dcc, n_obs, n_strains), dtype=bool)
    k = np.full(B, -1, dtype=np.int64)
    calls = []
    import daycare_replay
    ok = daycare_replay.row_ok(P, f, n_ind, n_strains, time_end)
    for i in range(B):
        if not ok[i]:
            continue

        class Counting:   # counts the lock-step transitions of the row
            def exponential(self, scale):
                calls.append(i)
                return rs.exponential(scale)

            def uniform(self, size):
                return rs.uniform(size=size)
        data[i] = dc.daycare(*P[i], n_dcc=n_dcc, n_ind=n_ind, n_strains=n_strains,
                             freq_strains_commun=f, n_obs=n_obs, time_end=time_end,
                             random_state=Counting())[0]
        k[i] = calls.count(i)
    if S is not None and d._addr(S):
        out = _summaries(data)
        out[k < 0] = np.nan
        d._mat(S, B, 4 * n_dcc, ldS)[:] = out
    if X is not None and d._addr(X):
        d._vec(X, data.size, np.uint8)[:] = data.reshape(-1)
    d._vec(K, B, np.int64)[:] = k


def daycare_summaries_f64(ctx, X, ld_b, ld_c, ld_i, ld_s, B, n_dcc, n_obs, n_strains, S, ldS,
                          stream):
    d._require(n_dcc >= 1 and n_obs >= 1 and 1 <= n_strains <= ops.DC_SUMM_STRAINS_MAX and
               ldS >= 4 * n_dcc, 'daycare_summaries: bad shape')
    if not B:
        return
    span = (B - 1) * ld_b + (n_dcc - 1) * ld_c + (n_obs - 1) * ld_i + (n_strains - 1) * ld_s + 1
    x = np.array(np.lib.stride_tricks.as_strided(d._vec(X, span, np.uint8),
                                                 (B, n_dcc, n_obs, n_strains),
                                                 (ld_b, ld_c, ld_i, ld_s))) != 0
    d._mat(S, B, 4 * n_dcc, ldS)[:] = _summaries(x)


def daycare_distance_f64(ctx, S, ldS, B, n_ss, n_dcc, obs_max, y, dist, stream):
    d._require(n_ss * n_dcc <= ops.DC_DIST_TERMS_MAX and ldS >= n_ss * n_dcc,
               'daycare_distance: bad shape')
    if not B:
        return
    # (n_ss, B, n_dcc) in C order, as np.stack lays out the reference's summaries
    s = np.ascontiguousarray(
        d._mat(S, B, n_ss * n_dcc, ldS).reshape(B, n_ss, n_dcc).transpose(1, 0, 2))
    om = d._vec(obs_max, n_ss)[:, None, None]
    yy = d._vec(y, n_ss * n_dcc).reshape(n_ss, 1, n_dcc)
    with np.errstate(all='ignore'):
        x = np.sort(s / om, axis=2)
        d._vec(dist, B)[:] = np.sum(np.abs(x - yy), axis=(0, 2)) / (n_ss * n_dcc)


TABLE = {'elfi_b200_' + f.__name__: f
         for f in (sim_daycare_f64, daycare_summaries_f64, daycare_distance_f64)}
