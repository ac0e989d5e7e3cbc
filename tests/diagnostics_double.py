"""NumPy restatement of the summary-selection entry points of include/elfi_b200.h
(elfi_b200_subset_distance_f64, elfi_b200_knn_entropy_f64, elfi_b200_mrsse_f64) and their CPU test
double -- TEST INFRASTRUCTURE ONLY.

`subset_distance` is SciPy's cdist on each combination's concatenated columns, `select` the first n
rows of a stable argsort by distance (NaN last: the order Rejection's batch-by-batch merge keeps),
`knn_radii` cKDTree's k-th distances and `mrsse` the reference's mean root sum of squared errors.
`TABLE` routes the three entry points here on top of tests/abi_double.py (through
`abi_double.install`), so the unmodified TwoStageSelection host code runs without a GPU.
"""
import numpy as np
from scipy.spatial import cKDTree
from scipy.spatial.distance import cdist

import abi_double as d

METRICS = ('euclidean', 'sqeuclidean', 'cityblock', 'chebyshev')


def subset_distance(S, obs, combinations, metric):
    """(C, B): cdist of the concatenated column ranges (col, width) of each combination."""
    S = np.asarray(S, dtype=np.float64)
    obs = np.asarray(obs, dtype=np.float64).reshape(-1)
    out = np.empty((len(combinations), S.shape[0]))
    for c, comb in enumerate(combinations):
        cols = np.concatenate([np.arange(col, col + w) for col, w in comb])
        out[c] = cdist(S[:, cols], obs[None, cols], metric)[:, 0]
    return out


def select(dist, n):
    """Row indices of the n smallest distances, ties in row order, NaN last."""
    return np.argsort(dist, kind='stable')[:n]


def knn_radii(X, k):
    """R[i] = cKDTree(X).query(X[i], k)[0][-1] (diagnostics.py:242-245)."""
    X = np.asarray(X, dtype=np.float64)
    tree = cKDTree(X)
    return np.array([np.atleast_1d(tree.query(x, k=k)[0])[-1] for x in X])


def mrsse(T, P):
    """diagnostics.py:284-289."""
    total = 0
    for p in P:
        total += np.sqrt(np.linalg.norm(T - p) ** 2)
    return total / len(P)


def subset_distance_f64(ctx, metric, S, ldS, B, W, obs, ranges, comb, C, d_out, ld_out, stream):
    d._require(1 <= W <= 512 and ldS >= W and 0 <= B < 2 ** 31 and 1 <= C < 2 ** 24 and
               ld_out >= B, 'subset_distance: bad shape')
    d._require(0 <= metric <= 3, 'subset_distance: bad metric')
    off = d._vec(comb, C + 1, np.int32)
    rg = d._mat(ranges, int(off[-1]), 2, dtype=np.int32)
    combs = [[tuple(rg[g]) for g in range(off[c], off[c + 1])] for c in range(C)]
    if not B:
        return
    d._mat(d_out, C, B, ld_out)[:] = subset_distance(d._mat(S, B, W, ldS), d._vec(obs, W), combs,
                                                     METRICS[metric])


def knn_entropy_f64(ctx, X, ldX, C, n, q, k, R, logsum, stream):
    d._require(1 <= q <= 16 and ldX >= q and 1 <= k <= 32 and 1 <= n <= 2 ** 20 and
               1 <= C < 2 ** 16, 'knn_entropy: bad shape')
    pts = d._mat(X, C * n, q, ldX)
    out = d._mat(R, C, n)
    for c in range(C):
        out[c] = knn_radii(pts[c * n:(c + 1) * n], k)
    with np.errstate(divide='ignore'):
        d._vec(logsum, C)[:] = np.log(out).sum(axis=1)


def mrsse_f64(ctx, T, ldT, C, n, q, P, ldP, m, out, stream):
    d._require(1 <= q <= 16 and ldT >= q and ldP >= q and n >= 1 and m >= 1 and C >= 1,
               'mrsse: bad shape')
    pts = d._mat(T, C * n, q, ldT)
    closest = np.array(d._mat(P, m, q, ldP))
    d._vec(out, C)[:] = [mrsse(pts[c * n:(c + 1) * n], closest) for c in range(C)]


TABLE = {'elfi_b200_' + f.__name__: f for f in (subset_distance_f64, knn_entropy_f64, mrsse_f64)}
