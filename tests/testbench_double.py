"""NumPy restatements of the segmented entry points of include/elfi_b200.h
(elfi_b200_dist_seg_f64, elfi_b200_topn_merge_seg_f64) and their CPU test double -- TEST
INFRASTRUCTURE ONLY.

`dist_seg` measures segment r of S against observed row r with the oracle's cdist restatements;
`topn_merge_seg` ranks each segment's [A_r; B_r] with a stable argsort (NaN last) and keeps the
n_keep smallest rows of every output.  `TABLE` routes both entry points here on top of
tests/abi_double.py (through `abi_double.install`), so the lock-step Testbench runs
without a GPU.
"""
import numpy as np

import abi_double as d
import elfi_oracle as o

METRIC_NAMES = {0: 'euclidean', 1: 'sqeuclidean', 2: 'cityblock', 3: 'chebyshev', 4: 'minkowski'}


def dist_seg(S, obs, metric='euclidean', p=2.0):
    """d (R B,) of S (R B, D) against obs (R, D), segment by segment."""
    S = np.asarray(S, dtype=np.float64)
    obs = np.atleast_2d(np.asarray(obs, dtype=np.float64))
    R = obs.shape[0]
    B = S.shape[0] // R
    out = np.empty(R * B)
    for r in range(R):
        X = np.ascontiguousarray(S[r * B:(r + 1) * B])
        if metric == 'euclidean':
            out[r * B:(r + 1) * B] = o.cdist_euclid(X, obs[r])
        else:
            out[r * B:(r + 1) * B] = o.cdist_metric(X, obs[r], metric, p)
    return out


def topn_merge_seg(A, B, keysA, keysB, n_keep):
    """Lists of (R, rows, w) arrays and (R, rows) keys -> list of (R, n_keep, w) arrays."""
    R = keysB.shape[0]
    outs = []
    orders = [np.argsort(np.concatenate([keysA[r], keysB[r]]), kind='stable')[:n_keep]
              for r in range(R)]
    for a, b in zip(A, B):
        outs.append(np.stack([np.concatenate([a[r], b[r]])[orders[r]] for r in range(R)]))
    return outs


def _seg(p, R, rows, width, ld, seg):
    """(R, rows, width) strided view over host memory."""
    if R == 0 or rows == 0:
        return np.empty((R, rows, width))
    span = (R - 1) * seg + (rows - 1) * ld + width
    flat = d._vec(p, span)
    return np.lib.stride_tricks.as_strided(flat, (R, rows, width), (8 * seg, 8 * ld, 8))


def dist_seg_f64(ctx, metric, pexp, S, ldS, R, B, D, obs, ld_obs, d_out, stream):
    d._require(metric in METRIC_NAMES, 'dist_seg: unknown metric code {}'.format(metric))
    d._require(R >= 1 and B >= 0 and D >= 1 and ldS >= D and ld_obs >= D, 'dist_seg: bad shape')
    d._require(R * B < 2 ** 31, 'dist_seg: R * B must fit int32')
    if not B:
        return
    X = np.array(d._mat(S, R * B, D, ldS))
    Y = np.array(d._mat(obs, R, D, ld_obs))
    d._vec(d_out, R * B)[:] = dist_seg(X, Y, METRIC_NAMES[metric], pexp)


def topn_merge_seg_f64(ctx, R, keysA, ld_keysA, seg_keysA, nA, keysB, ld_keysB, seg_keysB, nB,
                       n_keep, n_out, A_host, ldA_host, segA_host, B_host, ldB_host, segB_host,
                       width_host, dst_host, ld_dst_host, seg_dst_host, stream):
    d._require(R >= 1 and nA >= 0 and nB >= 0 and 0 <= n_keep <= nA + nB,
               'topn_merge_seg: bad sizes')
    d._require(R * (nA + nB) < 2 ** 31, 'topn_merge_seg: R * (nA + nB) must fit int32')
    if not (nA + nB and n_keep):
        return
    ka = _seg(keysA, R, nA, 1, ld_keysA, seg_keysA)[:, :, 0] if nA else np.empty((R, 0))
    kb = _seg(keysB, R, nB, 1, ld_keysB, seg_keysB)[:, :, 0] if nB else np.empty((R, 0))
    m = max(n_out, 1)
    pa, la, sa = (d._vec(A_host, m, np.uint64), d._vec(ldA_host, m, np.int64),
                  d._vec(segA_host, m, np.int64))
    pb, lb, sb = (d._vec(B_host, m, np.uint64), d._vec(ldB_host, m, np.int64),
                  d._vec(segB_host, m, np.int64))
    wd = d._vec(width_host, m, np.int64)
    pd, ld, sd = (d._vec(dst_host, m, np.uint64), d._vec(ld_dst_host, m, np.int64),
                  d._vec(seg_dst_host, m, np.int64))
    A, Bs = [], []
    for k in range(n_out):
        w = int(wd[k])
        A.append(np.array(_seg(int(pa[k]), R, nA, w, int(la[k]), int(sa[k]))) if nA
                 else np.empty((R, 0, w)))
        Bs.append(np.array(_seg(int(pb[k]), R, nB, w, int(lb[k]), int(sb[k]))) if nB
                  else np.empty((R, 0, w)))
    for k, top in enumerate(topn_merge_seg(A, Bs, ka, kb, n_keep)):
        w = int(wd[k])
        _seg(int(pd[k]), R, n_keep, w, int(ld[k]), int(sd[k]))[:] = top


TABLE = {'elfi_b200_dist_seg_f64': dist_seg_f64,
         'elfi_b200_topn_merge_seg_f64': topn_merge_seg_f64}
