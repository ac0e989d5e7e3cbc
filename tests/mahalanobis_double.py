"""NumPy restatement of the Mahalanobis distance of include/elfi_b200.h
(elfi_b200_dist_mahalanobis_thr_f64) and its CPU test double -- TEST INFRASTRUCTURE ONLY.

`cdist_mahalanobis` replays the kernel's order of operations with one NumPy operation per rounding:
for each row, u = S_i - obs, t_r = TS_c(VI[r, c] * u_c) over row r of VI, q = TS_r(u_r * t_r) and
d = sqrt(q), where TS is the two-sum order of SciPy's compiled loops (the one 'seuclidean' follows):
one running sum over the even and one over the odd positions of the first D - D%2 terms, added left
to right, then their sum, then the last term when D is odd.  NumPy's elementwise multiply and add
round once each, so nothing here contracts into an FMA.  `TABLE` routes the entry point here on top
of tests/abi_double.py (through `abi_double.install`), so the unmodified host code runs without a
GPU.
"""
import numpy as np

import abi_double as d

D_MAX = 192


def two_sum(terms):
    """TS over the last axis of `terms`: even and odd running sums, their sum, the odd last term."""
    n = terms.shape[-1]
    even = np.zeros(terms.shape[:-1])
    odd = np.zeros(terms.shape[:-1])
    for j in range(0, n - n % 2, 2):
        even = even + terms[..., j]
        odd = odd + terms[..., j + 1]
    s = even + odd
    return s + terms[..., n - 1] if n % 2 else s


def cdist_mahalanobis(S, obs, VI):
    """cdist(S, obs (1, D), 'mahalanobis', VI=VI) flattened to (B,), in the kernel's order."""
    S = np.asarray(S, dtype=np.float64)
    VI = np.asarray(VI, dtype=np.float64)
    u = S - np.asarray(obs, dtype=np.float64).reshape(1, -1)
    out = np.empty(len(u))
    step = max(1, (1 << 22) // VI.size)            # rows per chunk of (rows, D, D) products
    with np.errstate(invalid='ignore'):
        for i in range(0, len(u), step):
            uc = u[i:i + step]
            # t[i, r] = TS_c(VI[r, c] * u[i, c]): every r at once, each summed over c in order
            t = two_sum(VI[None, :, :] * uc[:, None, :])
            out[i:i + step] = np.sqrt(two_sum(uc * t))
    return out


def dist_mahalanobis_thr_f64(ctx, S, ldS, B, D, obs, VI, thr_host, d_out, acc_idx, n_acc, stream):
    d._require(d._addr(VI), 'dist_mahalanobis: VI is NULL')
    d._require(1 <= D <= D_MAX, 'dist_mahalanobis: D={} outside [1, {}]'.format(D, D_MAX))
    dist = cdist_mahalanobis(d._mat(S, B, D, ldS), d._vec(obs, D), d._mat(VI, D, D)) \
        if B else np.empty(0)
    if B:
        d._vec(d_out, B)[:] = dist
    thr = d._vec(thr_host, 1)
    if thr is not None:
        idx = d.o.accept_indices(dist, thr) if B else np.empty(0, dtype=np.int32)
        if d._addr(acc_idx):
            d._vec(acc_idx, max(B, 1), np.int32)[:len(idx)] = idx
        if d._addr(n_acc):
            d._vec(n_acc, 1, np.int64)[0] = len(idx)


TABLE = {'elfi_b200_dist_mahalanobis_thr_f64': dist_mahalanobis_thr_f64}
