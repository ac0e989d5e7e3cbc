"""NumPy restatement of the regression-adjustment entry points of include/elfi_b200.h
(elfi_b200_regadj_mask_f64, _moments_f64, _adjust_f64) and their CPU test double -- TEST
INFRASTRUCTURE ONLY.

`linear_adjust` states the whole device path with NumPy: the row masks, the groups (parameters
without a non-finite value on rows with finite summaries share one group, any other parameter has
its own), the count, means and centred moments of [S - o | theta_g] over a group's rows, the
device's solve rule (eigh of the q x q block, eigenvalues above tol^2 lambda_max, minimum-norm
solution) and the ordered adjusted columns.  `TABLE` routes the three entry points here on top
of tests/abi_double.py (through `abi_double.install`), so the unmodified host code
runs without a GPU.
"""
import numpy as np

import abi_double as d

D_MAX = 256


def row_mask(S, o):
    """Rows whose regressors S - o are all finite."""
    with np.errstate(invalid='ignore', over='ignore'):
        return np.isfinite(S - o).all(axis=1)


def groups(S, T, o):
    """[(columns, sel)] in the device's order: the shared group (sel = -1) first, if any."""
    rows = row_mask(S, o)
    bad = [int(np.sum(rows & ~np.isfinite(T[:, k]))) for k in range(T.shape[1])]
    shared = [k for k, b in enumerate(bad) if b == 0]
    return ([(shared, -1)] if shared else []) + [([k], k) for k, b in enumerate(bad) if b]


def members(S, T, o, sel):
    rows = row_mask(S, o)
    return rows if sel < 0 else rows & np.isfinite(T[:, sel])


def moments(S, T, o, cols, sel):
    """n_g, the means (d,) and the centred cross-products (d, d) of [S - o | T[:, cols]]."""
    m = members(S, T, o, sel)
    Z = np.column_stack([S[m] - o, T[m][:, cols]])
    n = int(m.sum())
    mean = Z.mean(axis=0) if n else np.full(Z.shape[1], np.nan)
    Zc = Z - mean if n else Z
    return n, mean, Zc.T @ Zc


def solve(M, q, n, tol=1e-6):
    """The device's solve rule (ops._regadj_solve, restated)."""
    A, B = M[:q, :q], M[:q, q:]
    w, V = np.linalg.eigh(A)
    keep = w > tol ** 2 * w[-1] if w[-1] > 0 else np.zeros(q, dtype=bool)
    coef = V[:, keep] @ np.diag(1.0 / w[keep]) @ V[:, keep].T @ B
    singular = np.sqrt(np.clip(np.sort(w)[::-1], 0, None))[:min(n, q)]
    return coef, int(keep.sum()), singular


def linear_adjust(S, T, o, tol=1e-6):
    """(adjusted, fits) as ops.linear_adjust returns them, on host arrays."""
    S = np.asarray(S, dtype=np.float64)
    T = np.asarray(T, dtype=np.float64)
    o = np.asarray(o, dtype=np.float64).reshape(-1)
    p, q = T.shape[1], S.shape[1]
    adjusted, fits = [None] * p, [None] * p
    for cols, sel in groups(S, T, o):
        n, mean, M = moments(S, T, o, cols, sel)
        if n == 0:
            raise ValueError('no finite row (n_samples = 0)')
        coef, rank, singular = solve(M, q, n, tol)
        intercept = mean[q:] - mean[:q] @ coef
        m = members(S, T, o, sel)
        X = S[m] - o
        for kk, k in enumerate(cols):
            adjusted[k] = T[m, k] - X @ coef[:, kk]
            fits[k] = dict(coef=coef[:, kk], intercept=float(intercept[kk]), rank=rank,
                           singular=singular, n_rows=n)
    return adjusted, fits


# ------------------------------------------------------------------------------ entry points
def _shape_ok(N, q, p, ldS, ldT):
    d._require(q >= 1 and p >= 1 and q + p <= D_MAX and 1 <= N < 2 ** 31 and ldS >= q and
               ldT >= p, 'regadj: bad shape')


def _inputs(S, ldS, N, q, obs, T, ldT, p):
    return (np.array(d._mat(S, N, q, ldS)), np.array(d._vec(obs, q)),
            np.array(d._mat(T, N, p, ldT)))


def _group(flags, N, T, cols_host, pg, sel, p):
    d._require(1 <= pg <= p and -1 <= sel < p, 'regadj: bad group')
    cols = [int(c) for c in d._vec(cols_host, pg, dtype=np.int32)]
    d._require(all(0 <= c < p for c in cols), 'regadj: bad column')
    m = np.array(d._vec(flags, N, dtype=np.uint8)) != 0
    if sel >= 0:
        m &= np.isfinite(T[:, sel])
    return cols, m


def regadj_mask_f64(ctx, S, ldS, N, q, obs, T, ldT, p, flags, counts, stream):
    _shape_ok(N, q, p, ldS, ldT)
    S, o, T = _inputs(S, ldS, N, q, obs, T, ldT, p)
    rows = row_mask(S, o)
    d._vec(flags, N, dtype=np.uint8)[:] = rows
    c = d._vec(counts, p + 1, dtype=np.int64)
    c[0] = rows.sum()
    c[1:] = [np.sum(rows & ~np.isfinite(T[:, k])) for k in range(p)]


def regadj_moments_f64(ctx, S, ldS, N, q, obs, T, ldT, p, flags, cols_host, pg, sel, mom, stream):
    _shape_ok(N, q, p, ldS, ldT)
    S, o, T = _inputs(S, ldS, N, q, obs, T, ldT, p)
    cols, m = _group(flags, N, T, cols_host, pg, sel, p)
    Z = np.column_stack([S[m] - o, T[m][:, cols]])
    dim = q + pg
    out = d._vec(mom, 1 + dim + dim * dim)
    n = int(m.sum())
    mean = Z.mean(axis=0) if n else np.full(dim, np.nan)
    out[0] = n
    out[1:1 + dim] = mean
    out[1 + dim:] = ((Z - mean).T @ (Z - mean) if n else np.zeros((dim, dim))).reshape(-1)


def regadj_adjust_f64(ctx, S, ldS, N, q, obs, T, ldT, p, flags, cols_host, pg, sel, dense, coef,
                      out, ld_out, stream):
    _shape_ok(N, q, p, ldS, ldT)
    d._require(dense in (0, 1) and ld_out >= (N if dense else 1), 'regadj: bad output')
    S, o, T = _inputs(S, ldS, N, q, obs, T, ldT, p)
    cols, m = _group(flags, N, T, cols_host, pg, sel, p)
    d._require(not dense or m.all(), 'regadj: dense with a row outside the group')
    C = np.array(d._mat(coef, q, pg))
    adj = T[m][:, cols] - (S[m] - o) @ C
    res = d._mat(out, pg, int(m.sum()), ld_out)
    res[:] = adj.T


TABLE = {'elfi_b200_regadj_mask_f64': regadj_mask_f64,
         'elfi_b200_regadj_moments_f64': regadj_moments_f64,
         'elfi_b200_regadj_adjust_f64': regadj_adjust_f64}
