"""CPU test double of the C ABI (include/elfi_b200.h) -- TEST INFRASTRUCTURE ONLY.

The product has no CPU path: elfi_b200 raises without a CUDA device.  To test the *host logic*
(operator wrappers in ops.py, the ElfiModel graph, Rejection / SMC state machines, the rank
sharding) on a machine without a GPU, the `cpu_double` fixture of tests/conftest.py swaps

  * elfi_b200._lib.call        -> the router `install` sets: every entry point restated on host
                                  pointers with NumPy + the oracle (same argument lists as the
                                  header), and
  * the allocation helpers of elfi_b200.device -> CPU torch tensors.

Nothing outside tests/ imports this module.  Entry points that the CPU tests do not need raise
ElfiB200Error so a test can never silently pass through an unimplemented call.
"""
import ctypes

import numpy as np
import torch

import elfi_oracle as o
from elfi_b200 import _lib

CALLS = []   # names of the entry points called (tests assert the expected kernels were reached)


def _addr(p):
    if p is None:
        return 0
    if isinstance(p, ctypes.c_void_p):
        return p.value or 0
    if isinstance(p, ctypes.Array):
        return ctypes.addressof(p)
    if isinstance(p, int):
        return p
    raise TypeError('unexpected pointer argument {!r}'.format(p))


def _mat(p, rows, cols, ld=None, dtype=np.float64):
    """(rows, cols) view with leading dimension ld over host memory; None for NULL."""
    a = _addr(p)
    if a == 0:
        return None
    rows, cols = int(rows), int(cols)
    ld = cols if ld is None else int(ld)
    item = np.dtype(dtype).itemsize
    if rows == 0 or cols == 0:
        return np.empty((rows, cols), dtype=dtype)
    nbytes = ((rows - 1) * ld + cols) * item
    buf = (ctypes.c_char * nbytes).from_address(a)
    flat = np.frombuffer(buf, dtype=dtype)
    return np.lib.stride_tricks.as_strided(flat, (rows, cols), (ld * item, item))


def _vec(p, n, dtype=np.float64):
    m = _mat(p, 1, n, dtype=dtype)
    return None if m is None else m[0]


def _require(cond, msg):
    if not cond:
        raise _lib.ElfiB200Error('cpu double: ' + msg)


# ------------------------------------------------------------------------------ entry points
def _distances(S, obs, W, K):
    d = np.empty((S.shape[0], K))
    for k in range(K):
        d[:, k] = o.cdist_euclid(np.ascontiguousarray(S), obs, w=None if W is None else W[k])
    return d


def dist_euclid_thr_f64(ctx, S, ldS, B, D, obs, W, K, thr_host, d_out, acc_idx, n_acc, stream):
    _require(K == 1 or _addr(W), 'K > 1 needs weights')
    S = _mat(S, B, D, ldS)
    d = _distances(S, _vec(obs, D), _mat(W, K, D), K) if B else np.empty((0, K))
    out = _mat(d_out, B, K)
    if B:
        out[:] = d
    thr = _vec(thr_host, K)
    if thr is not None:
        idx = o.accept_indices(d, thr) if B else np.empty(0, dtype=np.int32)
        if _addr(acc_idx):
            _vec(acc_idx, max(B, 1), np.int32)[:len(idx)] = idx
        if _addr(n_acc):
            _vec(n_acc, 1, np.int64)[0] = len(idx)


def dist_euclid_thr_dev_f64(ctx, S, ldS, B, D, obs, W, K, thr_dev, d_out, acc_idx, n_acc, stream):
    dist_euclid_thr_f64(ctx, S, ldS, B, D, obs, W, K, thr_dev, d_out, acc_idx, n_acc, stream)


def dist_euclid_mom_f64(ctx, S, ldS, B, D, obs, W, K, thr_host, thr_dev, d_out, acc_idx, n_acc, moments,
                        stream):
    thr = thr_host if _addr(thr_host) else thr_dev
    dist_euclid_thr_f64(ctx, S, ldS, B, D, obs, W, K, thr, d_out, acc_idx, n_acc, stream)
    colmoments_f64(ctx, S, ldS, B, D, moments, stream)


def accept_append_f64(ctx, acc_idx, n_acc, max_rows, n_src, src_host, ld_src_host, width_host, dst,
                      ld_dst, capacity, count, dropped, stream):
    _require(all(_addr(p) for p in (n_acc, src_host, ld_src_host, width_host, count)) and
             (_addr(dst) or capacity == 0), 'accept_append: NULL argument')
    _require(1 <= n_src <= 8, 'accept_append: 1..8 sources')
    _require(max_rows >= 0 and capacity >= 0, 'accept_append: bad shape')
    ptrs = _vec(src_host, n_src, np.uint64)
    lds = _vec(ld_src_host, n_src, np.int64)
    wid = _vec(width_host, n_src, np.int64)
    _require(all(ptrs) and all(wid >= 1) and all(lds >= wid), 'accept_append: bad source')
    _require(int(wid.sum()) <= ld_dst, 'accept_append: ld_dst < total width')
    if max_rows == 0:
        return
    n = int(_vec(n_acc, 1, np.int64)[0])
    cnt = _vec(count, 1, np.int64)
    rows = min(n, max(0, capacity - int(cnt[0])))
    idx = _vec(acc_idx, max(n, 1), np.int32)[:rows] if _addr(acc_idx) else np.arange(rows)
    out = _mat(dst, capacity, ld_dst)
    col = 0
    for k in range(n_src):
        if rows:
            nrows_src = int(idx.max()) + 1
            src = _mat(int(ptrs[k]), nrows_src, int(wid[k]), int(lds[k]))
            out[int(cnt[0]):int(cnt[0]) + rows, col:col + int(wid[k])] = src[idx]
        col += int(wid[k])
    if _addr(dropped):
        _vec(dropped, 1, np.int64)[0] += n - rows
    cnt[0] += rows


def rejection_batch_f64(ctx, S, ldS, B, D, obs, W, K, thr_host, thr_dev, d_out, acc_idx, n_acc, n_extra,
                        extra_host, ld_extra_host, width_extra_host, dst, ld_dst, capacity, count,
                        dropped, stream):
    _require(all(_addr(p) for p in (acc_idx, n_acc, d_out)), 'rejection_batch: NULL argument')
    _require(bool(_addr(thr_host)) != bool(_addr(thr_dev)),
             'rejection_batch: thresholds on the host OR on the device')
    _require(0 <= n_extra < 8, 'rejection_batch: 0..7 extra sources')
    thr = thr_host if _addr(thr_host) else thr_dev
    dist_euclid_thr_f64(ctx, S, ldS, B, D, obs, W, K, thr, d_out, acc_idx, n_acc, stream)
    ptrs = np.concatenate([[_addr(d_out)], _vec(extra_host, max(n_extra, 1), np.uint64)[:n_extra]]
                          ).astype(np.uint64)
    lds = np.concatenate([[K], _vec(ld_extra_host, max(n_extra, 1), np.int64)[:n_extra]]).astype(np.int64)
    wid = np.concatenate([[K], _vec(width_extra_host, max(n_extra, 1), np.int64)[:n_extra]]).astype(np.int64)
    accept_append_f64(ctx, acc_idx, n_acc, B, n_extra + 1, ctypes.c_void_p(ptrs.ctypes.data),
                      ctypes.c_void_p(lds.ctypes.data), ctypes.c_void_p(wid.ctypes.data), dst, ld_dst,
                      capacity, count, dropped, stream)


def dist_metric_thr_f64(ctx, metric, pexp, S, ldS, B, D, obs, thr_host, d_out, acc_idx, n_acc,
                        stream):
    name = {v: k for k, v in o.METRIC_CODES.items()}[metric]
    d = o.cdist_metric(np.ascontiguousarray(_mat(S, B, D, ldS)), _vec(obs, D), name, pexp) \
        if B else np.empty(0)
    if B:
        _vec(d_out, B)[:] = d
    thr = _vec(thr_host, 1)
    if thr is not None:
        idx = o.accept_indices(d, thr) if B else np.empty(0, dtype=np.int32)
        if _addr(acc_idx):
            _vec(acc_idx, max(B, 1), np.int32)[:len(idx)] = idx
        if _addr(n_acc):
            _vec(n_acc, 1, np.int64)[0] = len(idx)


def dist_seuclidean_thr_f64(ctx, S, ldS, B, D, obs, V, thr_host, d_out, acc_idx, n_acc, stream):
    _require(_addr(V), 'dist_seuclidean: V is NULL')
    d = o.cdist_seuclidean(np.ascontiguousarray(_mat(S, B, D, ldS)), _vec(obs, D), _vec(V, D)) \
        if B else np.empty(0)
    if B:
        _vec(d_out, B)[:] = d
    thr = _vec(thr_host, 1)
    if thr is not None:
        idx = o.accept_indices(d, thr) if B else np.empty(0, dtype=np.int32)
        if _addr(acc_idx):
            _vec(acc_idx, max(B, 1), np.int32)[:len(idx)] = idx
        if _addr(n_acc):
            _vec(n_acc, 1, np.int64)[0] = len(idx)


def summary_autocov_f64(ctx, X, ldX, B, n, lags_host, nlags, out, ld_out, stream):
    X = _mat(X, B, n, ldX)
    lags = _vec(lags_host, nlags, np.int32)
    out = _mat(out, B, nlags, ld_out)
    for c, lag in enumerate(lags):
        _require(1 <= lag < n, 'autocov: lag {} outside [1, n)'.format(lag))
        if B:
            out[:, c] = o.autocov(np.ascontiguousarray(X), int(lag))


def summary_meanvar_f64(ctx, X, ldX, B, n, out, ld_out, col_mean, col_var, stream):
    if not B:
        return
    X = _mat(X, B, n, ldX)
    mean, var = o.meanvar(np.ascontiguousarray(X))
    width = max(col_mean, col_var) + 1
    out = _mat(out, B, width, ld_out)
    if col_mean >= 0:
        out[:, col_mean] = mean
    if col_var >= 0:
        out[:, col_var] = var


def sort_pairs_f64(ctx, keys, n, keys_sorted, perm, stream):
    if not n:
        return
    k = _vec(keys, n)
    order = np.argsort(k, kind='stable')     # NaN last, ties by index: the ABI's contract
    if _addr(perm):
        _vec(perm, n, np.int32)[:] = order
    if _addr(keys_sorted):
        _vec(keys_sorted, n)[:] = k[order]


def gather_rows_f64(ctx, src, ld_src, idx, n, width, dst, ld_dst, stream):
    if not (n and width):
        return
    idx = _vec(idx, n, np.int32)
    src = _mat(src, int(idx.max()) + 1, width, ld_src)
    _mat(dst, n, width, ld_dst)[:] = src[idx]


def topn_merge_f64(ctx, keysA, ld_keysA, nA, keysB, ld_keysB, mapB, nB, n_keep, n_out, A_host, ldA_host,
                   B_host, ldB_host, width_host, dst_host, ld_dst_host, stream):
    _require(0 <= n_keep <= nA + nB, 'topn_merge: bad sizes')
    if not (nA + nB and n_keep):
        return
    mb = _vec(mapB, nB, np.int32).astype(np.int64) if _addr(mapB) and nB else np.arange(nB)
    ka = _mat(keysA, nA, 1, ld_keysA)[:, 0] if nA else np.empty(0)
    kb = _mat(keysB, int(mb.max()) + 1, 1, ld_keysB)[mb, 0] if nB else np.empty(0)
    order = np.argsort(np.concatenate([ka, kb]), kind='stable')[:n_keep]
    pa, la = _vec(A_host, max(n_out, 1), np.uint64), _vec(ldA_host, max(n_out, 1), np.int64)
    pb, lb = _vec(B_host, max(n_out, 1), np.uint64), _vec(ldB_host, max(n_out, 1), np.int64)
    wd = _vec(width_host, max(n_out, 1), np.int64)
    pd, ld = _vec(dst_host, max(n_out, 1), np.uint64), _vec(ld_dst_host, max(n_out, 1), np.int64)
    for k in range(n_out):
        w = int(wd[k])
        rows = []
        if nA:
            rows.append(_mat(int(pa[k]), nA, w, int(la[k])))
        if nB:
            rows.append(_mat(int(pb[k]), int(mb.max()) + 1, w, int(lb[k]))[mb])
        _mat(int(pd[k]), n_keep, w, int(ld[k]))[:] = np.concatenate(rows)[order]


def wquantile_f64(ctx, x, w, n, alpha, out, stream):
    _require(n >= 1 and 0.0 <= alpha <= 1.0, 'wquantile: bad arguments')
    x = _vec(x, n).copy()
    w = _vec(w, n)
    q = o.weighted_sample_quantile(x, alpha, None if w is None else w.copy())
    res = _vec(out, 2)
    res[0] = q
    res[1] = float(np.searchsorted(np.sort(x), q))


SM_COUNT = 132   # the multiprocessors colmoments_f64 sizes its grid by (an H100 SXM)


def colmoments_f64(ctx, S, ldS, B, D, out, stream):
    """colmoments_partial_kernel + colmoments_final_kernel (smc.cu) in their float64 order: shift
    by the first row; each block of R rows has 8 sequential chains (rows r0 + t, r0 + t + 8, ...),
    added t = 0 .. 7; the blocks are added in order; mean = x_0 + s1 / B, M2 = s2 - s1^2 / B.
    (The kernel's fma(d, d, s2) is a rounded product and add here: within the same bound.)"""
    S = np.ascontiguousarray(_mat(S, B, D, ldS))
    res = _mat(out, 2, D)
    colgroups = -(-D // 32)
    slabs = -(-(SM_COUNT * 8) // colgroups)
    rows = max(-(-B // slabs), 64)
    with np.errstate(invalid='ignore', over='ignore'):
        d = S - S[0]
        s1 = np.zeros(D)
        s2 = np.zeros(D)
        for r0 in range(0, B, rows):
            blk = d[r0:r0 + rows]
            b1 = np.zeros(D)
            b2 = np.zeros(D)
            for t in range(8):
                chain = blk[t::8]
                if len(chain):
                    b1 = b1 + np.cumsum(chain, axis=0)[-1]
                    b2 = b2 + np.cumsum(chain * chain, axis=0)[-1]
            s1 = s1 + b1
            s2 = s2 + b2
        res[0] = S[0] + s1 / B
        res[1] = s2 - s1 * s1 / B


def weighted_stats_f64(ctx, x, ldx, w, N, p, stats, stream):
    _require(N >= 1 and 1 <= p <= 16 and ldx >= p, 'weighted_stats: bad shape (p <= 16)')
    x = np.ascontiguousarray(_mat(x, N, p, ldx))
    w = np.ones(N) if not _addr(w) else _vec(w, N).copy()
    s = _vec(stats, 2 + 2 * p)
    s[0] = np.sum(w)
    s[1] = np.sum(w ** 2)
    with np.errstate(all='ignore'):
        s[2:2 + p] = np.average(x, weights=w, axis=0)
        s[2 + p:] = o.weighted_var(x, w)
        if np.count_nonzero(w) < 2:        # the header: V1 - V2 / V1 is exactly zero there
            s[2 + p:] = (w @ (x - s[2:2 + p]) ** 2) / 0.0


def gm_logpdf_f64(ctx, x, ldx, N, means, ldm, w, M, p, Linv_host, logdet, logq, stream):
    _require(N >= 0 and M >= 1 and 1 <= p <= 16 and ldx >= p and ldm >= p,
             'gm_logpdf: bad shape (p <= 16)')
    if N == 0:
        return
    # the oracle's density (SciPy's exp(lognorm - maha / 2), summed as plain densities), but
    # whitened with the Linv and logdet the caller passes, as the device does, and summed per
    # point so that a point's value does not depend on the rest of the batch
    x = np.ascontiguousarray(_mat(x, N, p, ldx))
    means = np.ascontiguousarray(_mat(means, M, p, ldm))
    Linv = np.array(_mat(Linv_host, p, p))
    weights = np.full(M, 1.0 / M) if not _addr(w) else _vec(w, M) / np.sum(_vec(w, M))
    lognorm = -0.5 * (p * np.log(2 * np.pi) + logdet)
    out = _vec(logq, N)
    b = max(1, (1 << 20) // M)
    for lo in range(0, N, b):
        z = (x[lo:lo + b, None, :] - means[None, :, :]) @ Linv.T
        with np.errstate(under='ignore'):
            dens = np.exp(lognorm - 0.5 * np.einsum('ijk,ijk->ij', z, z))
        with np.errstate(divide='ignore'):
            out[lo:lo + b] = np.log(np.sum(dens * weights, axis=1))


def gm_logpdf_mixed_f64(*args):
    gm_logpdf_f64(*args)


def smc_weights_f64(ctx, logprior, logq, n, w, stream):
    with np.errstate(all='ignore'):
        _vec(w, n)[:] = np.exp(_vec(logprior, n) - _vec(logq, n))


def rowsort_f64(ctx, X, ldX, B, n, out, ld_out, stream):
    _require(1 <= n <= 2048, 'rowsort: n outside [1, 2048]')
    if B:
        _mat(out, B, n, ld_out)[:] = np.sort(_mat(X, B, n, ldX), axis=1)


def kliep_fit_f64(ctx, x, ldx, Nx, y, ldy, Ny, p, wx, wy, sigma, n_basis, epsilon, max_iter,
                  abs_tol, conv_check_interval, alpha_out, result_host):
    xm = np.ascontiguousarray(_mat(x, Nx, p, ldx))
    ym = np.ascontiguousarray(_mat(y, Ny, p, ldy))
    alpha, max_ratio = o.kliep_fit(
        xm, ym, None if not _addr(wx) else _vec(wx, Nx).copy(),
        None if not _addr(wy) else _vec(wy, Ny).copy(), sigma=sigma, n=int(n_basis),
        epsilon=epsilon, max_iter=int(max_iter), abs_tol=abs_tol,
        conv_check_interval=int(conv_check_interval))
    _vec(alpha_out, n_basis)[:] = alpha
    out = _vec(result_host, 2)
    out[0] = max_ratio
    out[1] = -1.0   # the oracle does not count steps


# ---- BOLFI surrogate: SciPy restatement of the factor layout and the W-based arithmetic the
# header documents (var = k** - |W k|^2, T = W k, out = W^T T) ---------------------------------
def _gp_padded(n):
    return ((int(n) + 127) // 128) * 128


def _gp_kernel(A, B, kernel_var, lengthscale, bias_var):
    """k(A[i], B[j]) with r2 summed over coordinate differences, as gp.cu evaluates it (the
    expanded |a|^2 + |b|^2 - 2 a.b loses short distances to cancellation)."""
    r2 = np.zeros((len(A), len(B)))
    for d in range(A.shape[1]):
        diff = A[:, d, None] - B[None, :, d]
        r2 += diff * diff
    return kernel_var * np.exp(r2 * (-0.5 / lengthscale ** 2)) + bias_var


def gp_fit_f64(ctx, X, ldX, y, n, p, kernel_var, lengthscale, bias_var, noise_var, L, W, U, n_pad,
               alpha, info, stream):
    import scipy.linalg as sl
    _require(n >= 1 and p >= 1 and ldX >= p, 'gp_fit: bad shape')
    _require(n_pad == _gp_padded(n), 'gp_fit: n_pad must be {}'.format(_gp_padded(n)))
    Xm = np.ascontiguousarray(_mat(X, n, p, ldX))
    yv = _vec(y, n).copy()
    info_v = _vec(info, 1, np.int32)
    K = _gp_kernel(Xm, Xm, kernel_var, lengthscale, bias_var) + noise_var * np.eye(n)
    Lc, bad = sl.lapack.dpotrf(K, lower=1, clean=1)
    _require(bad >= 0, 'gp_fit: dpotrf argument error')
    # 1 + the index of the first non-positive pivot; some dpotrf builds do not flag NaN pivots,
    # which leave NaN on the diagonal
    nan_piv = np.flatnonzero(np.isnan(np.diagonal(Lc)[:bad - 1 if bad else n]))
    if nan_piv.size:
        bad = int(nan_piv[0]) + 1
    info_v[0] = bad
    if bad:
        return
    Lp = np.eye(n_pad)
    Lp[:n, :n] = Lc
    Wp = sl.solve_triangular(Lp, np.eye(n_pad), lower=True)
    _mat(L, n_pad, n_pad)[:] = Lp
    _mat(W, n_pad, n_pad)[:] = Wp
    _mat(U, n_pad, n_pad)[:] = Wp.T
    _vec(alpha, n)[:] = sl.cho_solve((Lc, True), yv)


def _gp_query(Xq, ldq, m, X, ldX, n, p, W, n_pad, kernel_var, lengthscale, bias_var):
    """(k = k(Xq, X) (m, n), W[:n, :n]) for the entry points that take a fitted W."""
    _require(m >= 0 and n >= 1 and p >= 1 and ldq >= p and ldX >= p, 'gp: bad shape')
    _require(n_pad == _gp_padded(n), 'gp: bad n_pad')
    Xm = np.ascontiguousarray(_mat(X, n, p, ldX))
    xq = np.ascontiguousarray(_mat(Xq, m, p, ldq))
    return _gp_kernel(xq, Xm, kernel_var, lengthscale, bias_var), np.array(_mat(W, n_pad, n_pad)[:n, :n])


def gp_predict_f64(ctx, Xq, ldq, m, X, ldX, n, p, W, n_pad, alpha, kernel_var, lengthscale,
                   bias_var, noise_add, beta, mean, var, acq, stream):
    k, Wn = _gp_query(Xq, ldq, m, X, ldX, n, p, W, n_pad, kernel_var, lengthscale, bias_var)
    if m == 0:
        return
    t = k.dot(Wn.T)
    mu = k.dot(_vec(alpha, n))
    v = (kernel_var + bias_var) - np.sum(t * t, axis=1)
    if _addr(mean):
        _vec(mean, m)[:] = mu
    if _addr(var):
        _vec(var, m)[:] = v + noise_add
    if _addr(acq):
        with np.errstate(invalid='ignore'):
            _vec(acq, m)[:] = o.lcbsc(mu, v, beta)


def gp_predict_grad_f64(ctx, Xq, ldq, m, X, ldX, n, p, W, U, n_pad, alpha, kernel_var,
                        lengthscale, bias_var, mean, var, grad_mean, grad_var, stream):
    """gpy_regression.py:206-218 with Ky^-1 = W^T W: t = W k, u = W^T t,
    grad_mean_d = sum_j dk_jd alpha_j, grad_var_d = -2 sum_j dk_jd u_j."""
    k, Wn = _gp_query(Xq, ldq, m, X, ldX, n, p, W, n_pad, kernel_var, lengthscale, bias_var)
    if m == 0:
        return
    xq = _mat(Xq, m, p, ldq)
    Xm = _mat(X, n, p, ldX)
    al = _vec(alpha, n)
    f = -0.5 / lengthscale ** 2
    t = k.dot(Wn.T)
    u = t.dot(Wn)
    dk = 2.0 * f * (xq[:, None, :] - Xm[None, :, :]) * (k - bias_var)[:, :, None]   # (m, n, p)
    if _addr(mean):
        _vec(mean, m)[:] = k.dot(al)
    if _addr(var):
        _vec(var, m)[:] = (kernel_var + bias_var) - np.sum(t * t, axis=1)
    if _addr(grad_mean):
        _mat(grad_mean, m, p)[:] = np.einsum('qjd,j->qd', dk, al)
    if _addr(grad_var):
        _mat(grad_var, m, p)[:] = -2.0 * np.einsum('qjd,qj->qd', dk, u)


def gp_whiten_f64(ctx, Xq, ldq, m, X, ldX, n, p, W, n_pad, kernel_var, lengthscale, bias_var, T,
                  ldT, stream):
    _require(ldT >= n, 'gp_whiten: bad shape')
    k, Wn = _gp_query(Xq, ldq, m, X, ldX, n, p, W, n_pad, kernel_var, lengthscale, bias_var)
    if m:
        _mat(T, m, n, ldT)[:] = k.dot(Wn.T)


def gp_apply_wt_f64(ctx, T, ldT, m, U, n_pad, n, out, ldo, stream):
    _require(m >= 0 and n >= 1 and ldT >= n and ldo >= n and n_pad >= n, 'gp_apply_wt: bad shape')
    if m:
        Un = _mat(U, n_pad, n_pad)[:n, :n]
        _mat(out, m, n, ldo)[:] = _mat(T, m, n, ldT).dot(Un.T)


def gp_cross_cov_f64(ctx, Xa, lda, ma, Ta, ldTa, Xb, ldb, mb, Tb, ldTb, n, p, kernel_var,
                     lengthscale, bias_var, cov, stream):
    if not (ma and mb):
        return
    xa = np.ascontiguousarray(_mat(Xa, ma, p, lda))
    xb = np.ascontiguousarray(_mat(Xb, mb, p, ldb))
    k = _gp_kernel(xb, xa, kernel_var, lengthscale, bias_var)
    g = _mat(Tb, mb, n, ldTb).dot(_mat(Ta, ma, n, ldTa).T)
    if (_addr(Xa), lda, ma, _addr(Ta), ldTa) == (_addr(Xb), ldb, mb, _addr(Tb), ldTb):
        # one point set: the device computes the same dot product for (a, b) and (b, a)
        g = np.tril(g) + np.tril(g, -1).T
    _mat(cov, mb, ma)[:] = k - g


def lcbsc_f64(ctx, mean, var, grad_mean, grad_var, m, p, beta, acq, grad_acq, stream):
    mu, v = _vec(mean, m), _vec(var, m)
    if _addr(acq):
        _vec(acq, m)[:] = o.lcbsc(mu, v, beta)
    if _addr(grad_acq):
        _mat(grad_acq, m, p)[:] = o.lcbsc_gradient(v[:, None], _mat(grad_mean, m, p),
                                                   _mat(grad_var, m, p), beta)


# ---- throughput mode: statistical stand-ins (NumPy RandomState instead of the device's Philox
# streams; same distributions, deterministic in (seed, offset), not sharding invariant) ---------
def _rs(seed, offset, salt=0):
    return np.random.RandomState((int(seed) * 1000003 + int(offset) * 7919 + salt) % (2 ** 32))


def prior_ma2_f64(ctx, B, seed, offset, mode, t1, t2, stream):
    from elfi_b200.examples import ma2 as ex
    rs = _rs(seed, offset, 1)
    if mode in (0, 1):
        _vec(t1, B)[:] = ex.CustomPrior1.rvs(2, size=B, random_state=rs)
    if mode in (0, 2):
        _vec(t2, B)[:] = ex.CustomPrior2.rvs(_vec(t1, B).copy(), 1, size=B, random_state=rs)


def logprior_ma2_f64(ctx, x, ldx, B, out, stream):
    from elfi_b200.examples import ma2 as ex
    xm = _mat(x, B, 2, ldx)
    with np.errstate(all='ignore'):
        _vec(out, B)[:] = ex.CustomPrior1.logpdf(xm[:, 0], 2) + ex.CustomPrior2.logpdf(
            xm[:, 1], xm[:, 0], 1)


def sim_ma2_f64(ctx, t1, t2, B, n_obs, seed, offset, X, ldX, S, ldS, stream):
    from elfi_b200.examples import ma2 as ex
    x = ex.MA2(_vec(t1, B).copy(), _vec(t2, B).copy(), n_obs=n_obs, batch_size=B,
               random_state=_rs(seed, offset, 2))
    if _addr(X):
        _mat(X, B, n_obs, ldX)[:] = x
    if _addr(S):
        out = _mat(S, B, 2, ldS)
        out[:, 0] = o.autocov(x, 1)
        out[:, 1] = o.autocov(x, 2)


def gm_cdf_f64(ctx, weights, N, cumw, stream):
    w = np.ones(N) if not _addr(weights) else _vec(weights, N)
    _vec(cumw, N)[:] = np.cumsum(w)


def gm_rvs_cdf_f64(ctx, means, ldm, cumw, N, p, Lchol_host, B, seed, offset, support, box_host, out,
                   ldo, stream):
    from elfi_b200.examples import ma2 as ex
    rs = _rs(seed, offset, 3)
    mu = _mat(means, N, p, ldm)
    w = np.diff(np.concatenate([[0.0], _vec(cumw, N)]))    # the weights back from their running sum
    L = _mat(Lchol_host, p, p)
    box = _vec(box_host, 2 * p) if support == 2 else None
    res = _mat(out, B, p, ldo)
    todo = np.arange(B)
    for _ in range(1000):
        comp = rs.choice(N, size=len(todo), p=w / w.sum())
        draw = mu[comp] + rs.randn(len(todo), p) @ L.T
        if support == 1:
            with np.errstate(all='ignore'):
                ok = np.isfinite(ex.CustomPrior1.logpdf(draw[:, 0], 2)
                                 + ex.CustomPrior2.logpdf(draw[:, 1], draw[:, 0], 1))
        elif support == 2:
            ok = np.all((draw >= box[:p]) & (draw <= box[p:]), axis=1)
        else:
            ok = np.ones(len(todo), dtype=bool)
        res[todo] = draw          # the last trial stays if no trial is accepted (as on the device)
        todo = todo[~ok]
        if not len(todo):
            break


def prior_gauss_f64(ctx, B, seed, offset, prm_host, mu, sigma, stream):
    import scipy.stats as ss
    prm = _vec(prm_host, 4)
    rs = _rs(seed, offset, 4)
    _vec(mu, B)[:] = prm[0] + prm[1] * (1.0 - rs.rand(B))       # (0, 1] like the device's u01
    _vec(sigma, B)[:] = ss.truncnorm.rvs(prm[2], prm[3], size=B, random_state=rs)


def logprior_gauss_f64(ctx, x, ldx, B, prm_host, out, stream):
    import scipy.stats as ss
    prm = _vec(prm_host, 4)
    xm = _mat(x, B, 2, ldx)
    with np.errstate(all='ignore'):
        _vec(out, B)[:] = ss.uniform.logpdf(xm[:, 0], prm[0], prm[1]) + ss.truncnorm.logpdf(
            xm[:, 1], prm[2], prm[3])


def sim_gauss_f64(ctx, mu, sigma, B, n_obs, seed, offset, Y, ldY, S, ldS, stream):
    y = _vec(mu, B)[:, None] + _vec(sigma, B)[:, None] * _rs(seed, offset, 5).randn(B, n_obs)
    if _addr(Y):
        _mat(Y, B, n_obs, ldY)[:] = y
    if _addr(S):
        out = _mat(S, B, 2, ldS)
        out[:, 0], out[:, 1] = o.meanvar(y)


def sim_gnk_f64(ctx, A, Bs, g, k, c, B, n_obs, seed, offset, Y, ldY, stream):
    z = _rs(seed, offset, 6).randn(B, n_obs)
    a, b, gg, kk = (_vec(v, B)[:, None] for v in (A, Bs, g, k))
    e = np.exp(-gg * z)
    _mat(Y, B, n_obs, ldY)[:] = a + b * (1 + c * ((1 - e) / (1 + e))) * (1 + z ** 2) ** kk * z


def logprior_box_f64(ctx, x, ldx, B, p, box_host, out, stream):
    box = _vec(box_host, 2 * p)
    xm = _mat(x, B, p, ldx)
    inside = np.all((xm >= box[:p]) & (xm <= box[:p] + box[p:]), axis=1)
    _vec(out, B)[:] = np.where(inside, -np.sum(np.log(box[p:])), -np.inf)


_TABLE = {'elfi_b200_' + f.__name__: f for f in (
    dist_euclid_thr_f64, dist_euclid_thr_dev_f64, dist_euclid_mom_f64, accept_append_f64, rejection_batch_f64, dist_metric_thr_f64, dist_seuclidean_thr_f64, topn_merge_f64, summary_autocov_f64, summary_meanvar_f64,
    sort_pairs_f64, gather_rows_f64, wquantile_f64, colmoments_f64,
    weighted_stats_f64, gm_logpdf_f64, gm_logpdf_mixed_f64, smc_weights_f64, rowsort_f64, kliep_fit_f64, gp_fit_f64,
    gp_predict_f64, gp_predict_grad_f64, gp_whiten_f64, gp_apply_wt_f64, gp_cross_cov_f64, lcbsc_f64, prior_ma2_f64, logprior_ma2_f64, sim_ma2_f64,
    gm_cdf_f64, gm_rvs_cdf_f64, prior_gauss_f64, logprior_gauss_f64, sim_gauss_f64, sim_gnk_f64, logprior_box_f64)}


# ------------------------------------------------------------------------------ device.py side
class DeviceTensor(torch.Tensor):
    """A CPU tensor that behaves like a CUDA tensor where the two differ for host code: it cannot
    be converted to NumPy implicitly (np.asarray / .numpy() raise, as they do for cuda tensors;
    .cpu() gives the plain tensor back) and it cannot be mixed with plain host tensors in torch
    operations (0-dim tensors excepted, as on the device).  This makes the CPU-double tests fail
    where the same code would fail on the GPU."""

    @staticmethod
    def wrap(t):
        return t if isinstance(t, DeviceTensor) else t.as_subclass(DeviceTensor)

    def __array__(self, *args, **kwargs):
        raise TypeError("can't convert cuda:0 device type tensor to numpy. Use Tensor.cpu() to "
                        "copy the tensor to host memory first. (cpu double)")

    def numpy(self, *args, **kwargs):
        return self.__array__()

    def cpu(self, *args, **kwargs):
        return self.as_subclass(torch.Tensor)

    def cuda(self, *args, **kwargs):
        return self

    @property
    def is_cuda(self):
        return True

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        name = getattr(func, '__name__', '')
        if name not in _MIX_OK:
            for a in _flatten(args) + _flatten(tuple(kwargs.values())):
                if isinstance(a, torch.Tensor) and not isinstance(a, DeviceTensor) and a.dim() > 0:
                    raise RuntimeError("Expected all tensors to be on the same device, but found at "
                                       "least two devices, cuda:0 and cpu! (cpu double, in {})"
                                       .format(name))
        return super().__torch_function__(func, types, args, kwargs)


_MIX_OK = {'__get__', '__set__', 'as_subclass', 'cpu', 'data_ptr', '__repr__', '__str__',
           '__format__', '__reduce_ex__', '__deepcopy__', 'all_gather_into_tensor'}


def _flatten(items):
    out = []
    for it in items:
        if isinstance(it, (list, tuple)):
            out += _flatten(it)
        else:
            out.append(it)
    return out


def install(monkeypatch, *tables):
    """Patch elfi_b200._lib.call and the allocation helpers of elfi_b200.device (CPU tensors that
    are as strict as CUDA tensors, see DeviceTensor).  Each of `tables` (entry point name ->
    restatement, the TABLE of a tests/*_double.py module) takes precedence over the ones before
    it and over this module's own; the tables are read at call time."""
    routes = tables[::-1] + (_TABLE,)

    def call(name, *args):
        """Stand-in for elfi_b200._lib.call: same names, same argument lists, host pointers."""
        fn = next((t[name] for t in routes if name in t), None)
        if fn is None:
            raise _lib.ElfiB200Error('cpu double: {} is not emulated (device-only entry point)'
                                     .format(name))
        if len(args) != len(_lib.SIGNATURES[name]):
            raise TypeError('{} takes {} arguments, got {}'.format(name, len(_lib.SIGNATURES[name]),
                                                                   len(args)))
        CALLS.append(name)
        fn(*args)
        return 0

    from elfi_b200 import device as dev
    from elfi_b200 import samplers

    def to_device(x, dtype=torch.float64):
        if isinstance(x, torch.Tensor):
            t = x if x.dtype == dtype else x.to(dtype)
            return DeviceTensor.wrap(t.contiguous())
        return DeviceTensor.wrap(
            torch.from_numpy(np.ascontiguousarray(x, dtype=dev._np_dtype(dtype)).copy()))

    gather = samplers.Comm.all_gather_rows

    def all_gather_rows(self, t):   # gloo works on plain tensors; the result is on "the device"
        out = gather(self, t.as_subclass(torch.Tensor) if isinstance(t, DeviceTensor) else t)
        return DeviceTensor.wrap(out) if isinstance(out, torch.Tensor) else out
    monkeypatch.setattr(samplers.Comm, 'all_gather_rows', all_gather_rows)

    monkeypatch.setattr(_lib, 'call', call)
    monkeypatch.setattr(dev, 'require_cuda', lambda: None)
    monkeypatch.setattr(dev, 'context', lambda device=None: ctypes.c_void_p(1))
    monkeypatch.setattr(dev, 'stream_ptr', lambda: ctypes.c_void_p(0))
    monkeypatch.setattr(dev, 'synchronize', lambda: None)
    monkeypatch.setattr(dev, 'is_device_array', lambda x: isinstance(x, DeviceTensor))
    monkeypatch.setattr(dev, 'to_device', to_device)
    monkeypatch.setattr(dev, 'empty', lambda shape, dtype=torch.float64:
                        DeviceTensor.wrap(torch.empty(shape, dtype=dtype)))
    monkeypatch.setattr(dev, 'zeros', lambda shape, dtype=torch.float64:
                        DeviceTensor.wrap(torch.zeros(shape, dtype=dtype)))
    monkeypatch.setattr(dev, 'ones', lambda shape, dtype=torch.float64:
                        DeviceTensor.wrap(torch.ones(shape, dtype=dtype)))
    monkeypatch.setattr(dev, 'full', lambda shape, value, dtype=torch.float64:
                        DeviceTensor.wrap(torch.full(shape, value, dtype=dtype)))
    del CALLS[:]
