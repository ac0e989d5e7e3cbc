"""CPU test double of the AR(1) entry point -- TEST INFRASTRUCTURE ONLY.

Extends tests/abi_double.py (through `abi_double.install`) with a restatement of
elfi_b200_sim_ar1_f64 on host pointers: the series is tests/ar1_replay.py (the kernel's Philox
streams and recursion, so the same rows as the device up to the last bits of the normals), the
distance and the accepted rows are the oracle's cdist and acceptance of exactly that series, as on
the device.
"""
import numpy as np

import abi_double as d
import ar1_replay
import elfi_oracle as o
from elfi_b200 import ops


def sim_ar1_f64(ctx, phi, B, n_obs, seed, offset, X, ldX, obs, thr_host, thr_dev, d_out, acc_idx,
                n_acc, stream):
    thr_p = thr_host if d._addr(thr_host) else thr_dev
    d._require(0 <= B <= ops.AR1_BATCH_MAX and 1 <= n_obs <= ops.AR1_NOBS_MAX and
               (not d._addr(X) or ldX >= n_obs), 'sim_ar1: bad shape')
    d._require(not (d._addr(thr_host) and d._addr(thr_dev)), 'sim_ar1: two thresholds')
    d._require(d._addr(obs) or not (d._addr(thr_p) or d._addr(d_out)),
               'sim_ar1: a distance needs obs')
    d._require(d._addr(thr_p) or not (d._addr(acc_idx) or d._addr(n_acc)),
               'sim_ar1: acc_idx requires thresholds')
    x = ar1_replay.sim_ar1(d._vec(phi, B), n_obs, seed, offset)[0] if B else np.empty((0, n_obs))
    if d._addr(X) and B:
        d._mat(X, B, n_obs, ldX)[:] = x
    if not d._addr(obs):
        return
    dist = o.cdist_euclid(x, d._vec(obs, n_obs)) if B else np.empty(0)
    if B:
        d._vec(d_out, B)[:] = dist.reshape(-1)
    thr = d._vec(thr_p, 1)
    if thr is not None:
        idx = o.accept_indices(dist.reshape(-1, 1), thr) if B else np.empty(0, dtype=np.int32)
        if d._addr(acc_idx):
            d._vec(acc_idx, max(B, 1), np.int32)[:len(idx)] = idx
        if d._addr(n_acc):
            d._vec(n_acc, 1, np.int64)[0] = len(idx)


TABLE = {'elfi_b200_' + f.__name__: f for f in (sim_ar1_f64,)}
