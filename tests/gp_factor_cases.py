"""Direct checks of the GP entry points of gp.cu against plain fp64 host arithmetic; the case
bodies shared by test_gp_factor_gpu.py (the device) and test_gp_factor_cpu_double.py (the CPU test
double, which shows that the checker itself is sound on LAPACK's factors).

The C ABI is called directly (not through GPyRegression) so that n, p, ldX, the hyper-parameters
and y are the test's.  Every output buffer is filled with NaN first: an entry that the header
promises and the kernel never writes fails every comparison.

Every bound is a rounding-error bound, u = 2^-53, C = 4 (the host products round as much as the
kernel's own).  A correct kernel meets it; a missing 4-wide k-step, a stale slab, a mis-ordered
look-ahead or a wrong tile of the inverse leaves errors of the order of the products themselves,
some 1e13 times larger.  The host evaluates k(a, b) itself from coordinate differences, as gp.cu
does; the two evaluations differ by at most about (p + 3) u |k| (p squares, exp, scale, bias),
which the bounds carry as a separate term.  References are built from the device's own W, U and
alpha where that isolates one kernel from the factorisation.

Coverage of the fit by shape.  n_pad = 128 ceil(n / 128); the Cholesky runs 64-wide panels
(potrf_diag_panel_kernel, the last block potrf_diag_kernel); launch_gemm sends a product to the
128 x 128 tile when it has >= 100 such tiles (mode 1 counts half + 1), else to the 64 x 64 tile.
The inverse W = L^-1 doubles s = 64, 128, ... < n_pad: nfull = n_pad // 2s full pairs go out as
one batched launch (grid.z = nfull) of two products of s x s tiles, and a partial pair with
s2 = n_pad - 2s nfull - s > 0 is launched on its own (s x s2, then s2 x s with the Ct store
into U).
  n = 1, 2, 3, 5            n_pad 128: one panel, then the last-block potrf_diag_kernel.
  n = 63 .. 129             n_pad 128 / 256: panel and padding edges.
  n = 255                   n_pad 256: every pair of the inverse is full.
  n = 257, 383, 641         n_pad 384, 384, 768: a partial pair (s2 = 128 at s = 256; s2 = 256
                            at s = 512) on the 64 x 64 tile.
  n = 1000                  n_pad 1024: every product on the 64 x 64 tile (at most 64 tiles).
  n = 2000, 2049            n_pad 2048, 2176: the trailing update of the first panels (below2 =
                            1920, 1856 at 2048) has 15^2 / 2 + 1 = 113 tiles -> 128 x 128, mode 1;
                            the inverse stays on the 64 x 64 tile (s = 1024: 64 tiles; 2176:
                            s2 = 128 at s = 2048, 16 tiles).
  n = 3900                  n_pad 3968: s = 2048 has no full pair and a partial pair s2 = 1920:
                            16 x 15 = 240 tiles on the 128 x 128 tile, including its Ct store
                            into U.  (s = 1024: one full pair, 64 tiles, and s2 = 896: 56.)
  n = 4097                  n_pad 4224: s = 1024 has two full pairs, 2 x 64 = 128 tiles: a
                            batched 128 x 128 launch with grid.z = 2; s = 2048 one full pair of
                            256 tiles; s = 4096 a partial pair s2 = 128 on the 64 x 64 tile.
If a tiling change moves these thresholds, the shapes above are the ones to revisit.
"""
import types

import numpy as np
import pytest
import scipy.linalg as sl
import torch

from elfi_b200 import _lib
from elfi_b200 import device as dev

U_RND = 2.0 ** -53
C = 4.0


def padded(n):
    return ((n + 127) // 128) * 128


def rbf_bias(A, B, s2, l, b):
    """k(A[i], B[j]) = s2 exp(-|A_i - B_j|^2 / (2 l^2)) + b, r2 from coordinate differences."""
    r2 = np.zeros((len(A), len(B)))
    for d in range(A.shape[1]):
        diff = A[:, d, None] - B[None, :, d]
        r2 += diff * diff
    return s2 * np.exp(r2 * (-0.5 / l ** 2)) + b


class Report:
    """Largest ratio err / (k u scale) per check; every check must stay within C (plus its
    kernel-evaluation term).  The whole report goes into the failure message."""

    def __init__(self, what):
        self.what, self.ratio, self.failed = what, {}, []

    def bound(self, name, err, scale, k, extra=0.0):
        err = np.asarray(err, dtype=float)
        scale = np.broadcast_to(np.asarray(scale, dtype=float), err.shape)
        tol = C * k * U_RND * scale + extra
        with np.errstate(divide='ignore', invalid='ignore'):
            r = np.where(scale > 0, err / (k * U_RND * scale), np.where(err == 0, 0.0, np.inf))
        self.ratio[name] = float(np.max(r)) if r.size else 0.0
        if not np.all(err <= tol):      # NaN fails
            self.failed.append(name)

    def exact(self, name, ok):
        if not ok:
            self.failed.append(name)

    def check(self):
        assert not self.failed, '{}: {} failed; ratios {}'.format(self.what, self.failed, self.ratio)
        return self.ratio


# ---------------------------------------------------------------------------- calls
def _rows(A, ld):
    """(rows, p) host array -> device buffer with leading dimension ld, NaN in the gap."""
    buf = np.full((A.shape[0], ld), np.nan)
    buf[:, :A.shape[1]] = A
    return dev.to_device(buf)


def fit(X, y, hyper, ldX=None):
    """elfi_b200_gp_fit_f64 on (X, y); hyper = (kernel_var, lengthscale, bias_var, noise_var)."""
    n, p = X.shape
    ldX = p if ldX is None else ldX
    n_pad = padded(n)
    assert int(_lib.load().elfi_b200_gp_padded_size(n)) == n_pad
    F = types.SimpleNamespace(X=X, y=y, hyper=hyper, n=n, p=p, n_pad=n_pad, Xd=_rows(X, ldX),
                              ldX=ldX, yd=dev.to_device(y))
    F.Ld, F.Wd, F.Ud = (dev.full((n_pad, n_pad), np.nan) for _ in range(3))
    F.alphad = dev.full((n,), np.nan)
    info = dev.full((1,), -1, dtype=torch.int32)
    _lib.call('elfi_b200_gp_fit_f64', dev.context(), dev.ptr(F.Xd), ldX, dev.ptr(F.yd), n, p,
              *hyper, dev.ptr(F.Ld), dev.ptr(F.Wd), dev.ptr(F.Ud), n_pad, dev.ptr(F.alphad),
              dev.ptr(info), dev.stream_ptr())
    F.info = int(dev.to_host(info)[0])
    F.L, F.W, F.U, F.alpha = (dev.to_host(t) for t in (F.Ld, F.Wd, F.Ud, F.alphad))
    return F


def predict(F, Q, noise_add=0.0, beta=None, ldq=None):
    m, p = Q.shape
    ldq = p if ldq is None else ldq
    s2, l, b, _ = F.hyper
    Qd = _rows(Q, ldq)
    mean, var, acq = (dev.full((m,), np.nan) for _ in range(3))
    _lib.call('elfi_b200_gp_predict_f64', dev.context(), dev.ptr(Qd), ldq, m,
              dev.ptr(F.Xd), F.ldX, F.n, p, dev.ptr(F.Wd), F.n_pad, dev.ptr(F.alphad), s2, l, b,
              noise_add, 0.0 if beta is None else beta, dev.ptr(mean), dev.ptr(var),
              dev.ptr(acq) if beta is not None else None, dev.stream_ptr())
    return dev.to_host(mean), dev.to_host(var), dev.to_host(acq)


def predict_grad(F, Q, n_pad=None):
    m, p = Q.shape
    s2, l, b, _ = F.hyper
    mean, var = dev.full((m,), np.nan), dev.full((m,), np.nan)
    gm, gv = dev.full((m, p), np.nan), dev.full((m, p), np.nan)
    Qd = _rows(Q, p + 2)
    _lib.call('elfi_b200_gp_predict_grad_f64', dev.context(), dev.ptr(Qd), p + 2, m,
              dev.ptr(F.Xd), F.ldX, F.n, p, dev.ptr(F.Wd), dev.ptr(F.Ud),
              F.n_pad if n_pad is None else n_pad, dev.ptr(F.alphad), s2, l, b, dev.ptr(mean),
              dev.ptr(var), dev.ptr(gm), dev.ptr(gv), dev.stream_ptr())
    return tuple(dev.to_host(t) for t in (mean, var, gm, gv))


def whiten(F, Q, ldT):
    """-> (device T (m, ldT), host copy)"""
    m, p = Q.shape
    s2, l, b, _ = F.hyper
    T = dev.full((m, ldT), np.nan)
    Qd = _rows(Q, p)
    _lib.call('elfi_b200_gp_whiten_f64', dev.context(), dev.ptr(Qd), p, m, dev.ptr(F.Xd),
              F.ldX, F.n, p, dev.ptr(F.Wd), F.n_pad, s2, l, b, dev.ptr(T), ldT, dev.stream_ptr())
    return T, dev.to_host(T)


def apply_wt(F, T, ldo):
    m, ldT = T.shape
    out = dev.full((m, ldo), np.nan)
    _lib.call('elfi_b200_gp_apply_wt_f64', dev.context(), dev.ptr(T), ldT, m, dev.ptr(F.Ud),
              F.n_pad, F.n, dev.ptr(out), ldo, dev.stream_ptr())
    return dev.to_host(out)


def cross_cov(F, A, TA, B, TB):
    s2, l, b, _ = F.hyper
    Ad = dev.to_device(A)
    Bd = Ad if B is A else dev.to_device(B)
    cov = dev.full((len(B), len(A)), np.nan)
    _lib.call('elfi_b200_gp_cross_cov_f64', dev.context(), dev.ptr(Ad), F.p, len(A), dev.ptr(TA),
              TA.shape[1], dev.ptr(Bd), F.p, len(B), dev.ptr(TB), TB.shape[1], F.n, F.p, s2, l, b,
              dev.ptr(cov), dev.stream_ptr())
    return dev.to_host(cov)


# ---------------------------------------------------------------------------- data
def data(n, p, cond, seed=0):
    """(X, y, hyper).  'well': lengthscale 0.2, noise 0.05.  'bad': lengthscale 2 on the unit
    cube and noise n (s2 + b) 1e-7, so cond(Ky) ~ 1e6 .. 1e7 once n is more than a few points."""
    rs = np.random.RandomState(seed + 7919 * n + 31 * p)
    X = rs.uniform(0.0, 1.0, (n, p))
    y = np.sin(3.0 * X).sum(axis=1) + 0.1 * rs.randn(n)
    s2, b = 1.0, 0.5
    if cond == 'well':
        return X, y, (s2, 0.2, b, 0.05)
    return X, y, (s2, 2.0, b, n * (s2 + b) * 1e-7)


FIT_SMALL = [(1, 1, 1), (2, 2, 5), (3, 5, 5), (5, 10, 13), (63, 1, 4), (64, 2, 2), (65, 5, 8),
             (127, 10, 10), (128, 2, 5), (129, 1, 1), (255, 5, 5), (257, 2, 5), (383, 10, 13),
             (641, 1, 4), (1000, 2, 2)]                     # (n, p, ldX), each well and bad
FIT_LARGE = [(2000, 5, 8, 'bad'), (2049, 2, 2, 'well'), (3900, 2, 5, 'well'),
             (4097, 10, 13, 'bad')]                          # once each: host products are O(n^3)


# ---------------------------------------------------------------------------- fit
def case_fit(n, p, ldX, cond):
    """Backward error of L, both inverse residuals, exact structure, alpha, log-determinant and
    determinism of one fit."""
    X, y, hyper = data(n, p, cond)
    F = fit(X, y, hyper, ldX)
    assert F.info == 0, F.info
    s2, l, b, noise = hyper
    n_pad = F.n_pad
    rep = Report('fit n={} p={} ldX={} {}'.format(n, p, ldX, cond))
    Ky = rbf_bias(X, X, s2, l, b) + noise * np.eye(n)
    kerr = (p + 3) * U_RND * np.abs(Ky)

    # exact structure: W lower with exact zeros above the diagonal, U = W^T, identity padding
    Lp = np.tril(F.L)
    eye = np.eye(n_pad - n)
    rep.exact('triu(W, 1) == 0', np.all(np.triu(F.W, 1) == 0))
    rep.exact('U == W^T', np.array_equal(F.U, F.W.T))
    for name, M in (('L', F.L), ('W', F.W), ('U', F.U)):
        rep.exact(name + ' padding', np.array_equal(M[n:, n:], eye) and np.all(M[n:, :n] == 0)
                  and np.all(M[:n, n:] == 0))
    rep.exact('diag(L) > 0', np.all(np.diagonal(F.L)[:n] > 0))

    # |L L^T - Ky| <= C (n + 1) u |L| |L^T|, lower triangle
    Lh = Lp[:n, :n]
    aL = np.abs(Lh)
    B = aL @ aL.T
    low = np.tril(np.ones((n, n), dtype=bool))
    rep.bound('L L^T - Ky', np.abs(Lh @ Lh.T - Ky)[low], B[low], n + 1, kerr[low])

    # inverse residuals on the padded matrices
    I = np.eye(n_pad)
    aW, aLp = np.abs(F.W), np.abs(Lp)
    rep.bound('W L - I', np.abs(F.W @ Lp - I), aW @ aLp, n)
    rep.bound('L W - I', np.abs(Lp @ F.W - I), aLp @ aW, n)

    # alpha against W^T (W y) from the device's own W (two matrix-vector products, each within
    # n u of |W| |.|, on both sides), and its residual
    Wn = F.W[:n, :n]
    ref = Wn.T @ (Wn @ y)
    aWn = np.abs(Wn)
    rep.bound('alpha - W^T W y', np.abs(F.alpha - ref), aWn.T @ (aWn @ np.abs(y)), n)
    rep.bound('Ky alpha - y', np.abs(Ky @ F.alpha - y), np.abs(Ky) @ np.abs(F.alpha) + np.abs(y),
              n, (p + 3) * U_RND * (np.abs(Ky) @ np.abs(F.alpha)))

    # log det, to first order: |d logdet| <= sum |Ky^-1| o |dKy|, with |dKy| <= C (n + 1) u |L||L^T|
    # from the factor, (p + 3) u |Ky| from the kernel evaluation, and Ky^-1 = W^T W
    sign, ref_ld = np.linalg.slogdet(Ky)
    assert sign > 0
    ld = 2.0 * np.sum(np.log(np.diagonal(F.L)[:n]))
    rep.bound('logdet', abs(ld - ref_ld), np.sum(np.abs(Wn.T @ Wn) * B), n + p + 4)

    # determinism: the look-ahead side stream (ev_panel / ev_rest) must not change a bit
    G = fit(X, y, hyper, ldX)
    rep.exact('bit-identical refit', all(np.array_equal(a.view(np.int64), c.view(np.int64))
                                         for a, c in ((F.L, G.L), (F.W, G.W), (F.U, G.U),
                                                      (F.alpha, G.alpha))))
    return rep.check()


# ---------------------------------------------------------------------------- prediction
PREDICT_N = [(256, 2), (257, 1), (130, 5), (383, 10)]      # n = 0, 1, 2, 3 (mod 4)
PREDICT_M = [1, 15, 16, 17, 160, 161, 1000, 32768, 32769]  # <= 160: trimv; 32769: two chunks


def _queries(F, m, seed):
    """m points: some training points (variance down at the noise), the rest uniform."""
    rs = np.random.RandomState(seed)
    k = min(F.n, m // 4)
    return np.vstack([F.X[:k], rs.uniform(-0.1, 1.1, (m - k, F.p))])


def _predict_refs(F, Q):
    s2, l, b, _ = F.hyper
    K = rbf_bias(Q, F.X, s2, l, b)
    Wn = F.W[:F.n, :F.n]
    T = K @ Wn.T
    S = np.abs(K) @ np.abs(Wn).T
    return K, T, S


def _check_predict(rep, tag, F, Q, mean, var, noise_add, refs):
    s2, l, b, _ = F.hyper
    K, T, S = refs
    n, p = F.n, F.p
    rep.bound(tag + ' mean', np.abs(mean - K @ F.alpha), np.abs(K) @ np.abs(F.alpha), n + p + 3)
    var_ref = (s2 + b) - np.sum(T * T, axis=1) + noise_add
    rep.bound(tag + ' var', np.abs(var - var_ref), np.sum(S * S, axis=1), n + 2 * (p + 3),
              C * U_RND * (s2 + b + abs(noise_add)))


def case_predict(n, p):
    """gp_predict_f64 on both paths (m <= 160: trimv; else the triangular-skip GEMM with its
    row-square epilogue, K rounded to (n + 3) & ~3) against K* alpha and kss - |W k|^2 built from
    the device's W and alpha; acq = mean - sqrt(beta var) bit for bit."""
    X, y, hyper = data(n, p, 'well', seed=1)
    F = fit(X, y, hyper, ldX=p + 3)
    rep = Report('predict n={} p={}'.format(n, p))
    beta = 2.7
    for m in PREDICT_M:
        Q = _queries(F, m, seed=m)
        refs = _predict_refs(F, Q)
        mean, var, acq = predict(F, Q, beta=beta, ldq=p + 1)
        _check_predict(rep, 'm={}'.format(m), F, Q, mean, var, 0.0, refs)
        with np.errstate(invalid='ignore'):
            rep.exact('m={} acq'.format(m), np.array_equal(acq, mean - np.sqrt(beta * var),
                                                           equal_nan=True))
        if m in (17, 1000):
            mean2, var2, _ = predict(F, Q, noise_add=0.125)
            _check_predict(rep, 'm={} noise'.format(m), F, Q, mean2, var2, 0.125, refs)
    # the two paths on the same 160 points
    Q = _queries(F, 320, seed=5)
    refs = _predict_refs(F, Q[:160])
    mg, vg, _ = predict(F, Q)
    mt, vt, _ = predict(F, Q[:160])
    _check_predict(rep, 'gemm', F, Q[:160], mg[:160], vg[:160], 0.0, refs)
    _check_predict(rep, 'trimv', F, Q[:160], mt, vt, 0.0, refs)
    return rep.check()


WHITEN_N = [(255, 2), (257, 3), (641, 1)]                  # straddle the 256-column slabs
WHITEN_M = [1, 4, 5, 8, 9, 16, 17, 33]                     # every MQ instance, 16-point chunks


def case_whiten_apply_wt(n, p):
    """gp_whiten_f64: T = W k over rows < n (ldT > n, nothing written beyond n);
    gp_apply_wt_f64: out = U[:n, :n] T, the upper path of gp_trimv_kernel."""
    X, y, hyper = data(n, p, 'well', seed=2)
    F = fit(X, y, hyper)
    rep = Report('whiten n={} p={}'.format(n, p))
    Wn, Un = F.W[:n, :n], F.U[:n, :n]
    for m in WHITEN_M:
        Q = _queries(F, m, seed=100 + m)
        K, Tref, S = _predict_refs(F, Q)
        Td, T = whiten(F, Q, ldT=n + 5)
        rep.bound('m={} T'.format(m), np.abs(T[:, :n] - Tref), S, n + p + 3)
        rep.exact('m={} T tail untouched'.format(m), np.all(np.isnan(T[:, n:])))
        out = apply_wt(F, Td, ldo=n + 3)
        rep.bound('m={} W^T T'.format(m), np.abs(out[:, :n] - T[:, :n] @ Un.T),
                  np.abs(T[:, :n]) @ np.abs(Un).T, n)
        rep.exact('m={} out tail untouched'.format(m), np.all(np.isnan(out[:, n:])))
    return rep.check()


GRAD_N = [(130, 5), (257, 1), (383, 10)]
GRAD_M = [1, 5, 16, 17]


def case_predict_grad(n, p):
    """gp_predict_grad_f64 against gpy_regression.py:211-218 on the host with the device's W and
    alpha: dk_jd = 2 f (x_d - X_jd) kx_j, grad_mean = dk^T alpha, grad_var = -2 dk^T W^T W k."""
    X, y, hyper = data(n, p, 'well', seed=3)
    F = fit(X, y, hyper)
    s2, l, b, _ = hyper
    f = -0.5 / l ** 2
    rep = Report('predict_grad n={} p={}'.format(n, p))
    Wn = F.W[:n, :n]
    aW = np.abs(Wn)
    for m in GRAD_M:
        Q = _queries(F, m, seed=200 + m)
        refs = _predict_refs(F, Q)
        K, T, S = refs
        mean, var, gm, gv = predict_grad(F, Q)
        _check_predict(rep, 'm={}'.format(m), F, Q, mean, var, 0.0, refs)
        kx = rbf_bias(Q, X, s2, l, 0.0)
        dx = 2.0 * f * (Q[:, None, :] - X[None, :, :])                  # (m, n, p)
        dk = dx * kx[:, :, None]
        u = T @ Wn
        D = np.abs(dx) * (np.abs(kx) + b)[:, :, None]                   # kq - b cancels to ~u kq
        umag = S @ aW
        rep.bound('m={} grad_mean'.format(m), np.abs(gm - np.einsum('qjd,j->qd', dk, F.alpha)),
                  np.einsum('qjd,j->qd', D, np.abs(F.alpha)), n + p + 6)
        rep.bound('m={} grad_var'.format(m), np.abs(gv + 2.0 * np.einsum('qjd,qj->qd', dk, u)),
                  2.0 * (np.einsum('qjd,qj->qd', D, np.abs(u))
                         + np.einsum('qjd,qj->qd', np.abs(dk), umag)), 2 * n + p + 6)
    return rep.check()


def case_predict_grad_checks_n_pad():
    """A wrong n_pad would read W with the wrong leading dimension: refused, and the context
    stays usable."""
    X, y, hyper = data(200, 2, 'well', seed=4)
    F = fit(X, y, hyper)
    Q = _queries(F, 5, seed=9)
    before = predict_grad(F, Q)
    for bad in (F.n_pad + 128, F.n_pad - 128):
        with pytest.raises(_lib.ElfiB200Error, match='n_pad'):
            predict_grad(F, Q, n_pad=bad)
    after = predict_grad(F, Q)
    for a, c in zip(before, after):
        assert np.array_equal(a, c)


CROSS_MA = [1, 10, 19, 28, 37, 46, 55]                      # 1 .. 7 (mod 8)


def case_cross_cov(n=257, p=2):
    """gp_cross_cov_f64 = k(a, b) - T_a . T_b from the device's T; exactly symmetric for a = b."""
    X, y, hyper = data(n, p, 'well', seed=6)
    F = fit(X, y, hyper)
    s2, l, b, _ = hyper
    rep = Report('cross_cov n={} p={}'.format(n, p))
    rs = np.random.RandomState(11)
    for mb in (2, 9):
        B = rs.uniform(0, 1, (mb, p))
        TBd, TB = whiten(F, B, ldT=n + 1)
        for ma in CROSS_MA:
            A = rs.uniform(0, 1, (ma, p))
            TAd, TA = whiten(F, A, ldT=n + 3)
            cov = cross_cov(F, A, TAd, B, TBd)
            k = rbf_bias(B, A, s2, l, b)
            G = TB[:, :n] @ TA[:, :n].T
            rep.bound('ma={} mb={}'.format(ma, mb), np.abs(cov - (k - G)),
                      np.abs(k) + np.abs(TB[:, :n]) @ np.abs(TA[:, :n]).T, n + p + 3)
    for ma in CROSS_MA:
        A = rs.uniform(0, 1, (ma, p))
        TAd, _ = whiten(F, A, ldT=n + 3)
        cov = cross_cov(F, A, TAd, A, TAd)
        rep.exact('ma={} symmetric'.format(ma), np.array_equal(cov, cov.T))
    return rep.check()


# ---------------------------------------------------------------------------- first bad pivot
PIVOT_CASES = [(350, j0, kind) for kind in ('dup', 'nan') for j0 in (1, 63, 64, 65, 200, 349)] + \
    [(100, 99, 'dup'), (100, 70, 'nan')]
# n = 350 (n_pad 384): j0 < 320 in potrf_diag_panel_kernel, 349 in the last block (320..383),
# as are 70 and 99 at n = 100 (n_pad 128, last block 64..127)


def pivot_data(n, j0, kind):
    """Points 1 apart on a grid, lengthscale 0.05: Ky = (1 + noise) I + 0.5 11^T up to 1e-87.
    'dup': point j0 repeats point j0 // 2 and noise = -0.01, so every pivot before j0 is ~1 and
    pivot j0 is 2 noise - noise^2 (Ky_prev^-1)_ii < 0.  'nan': row j0 of X is NaN."""
    X = np.stack([np.arange(n) % 20, np.arange(n) // 20], axis=1).astype(float)
    y = np.cos(np.arange(n, dtype=float))
    if kind == 'dup':
        X[j0] = X[j0 // 2]
        noise = -0.01
    else:
        X[j0, 1] = np.nan
        noise = 0.01
    return X, y, (1.0, 0.05, 0.5, noise)


def case_first_bad_pivot(n, j0, kind):
    """info = 1 + the index of the FIRST non-positive pivot, as LAPACK's dpotrf reports it, and
    GPyRegression._fit names that index.  dpotrf implementations differ on NaN pivots (the
    reference LAPACK flags them, OpenBLAS's does not), so the NaN cases compare with j0 + 1."""
    from elfi_b200.bo import JITTER, GPyRegression
    X, y, hyper = pivot_data(n, j0, kind)
    s2, l, b, noise = hyper
    F = fit(X, y, hyper)
    if kind == 'dup':
        Ky = rbf_bias(X, X, s2, l, b) + noise * np.eye(n)
        lapack = sl.lapack.dpotrf(Ky, lower=1)[1]
        assert lapack == j0 + 1, lapack
    assert F.info == j0 + 1, (F.info, j0 + 1)
    gp = GPyRegression(['a', 'b'], bounds={'a': (0, 20), 'b': (0, 20)})
    gp._X, gp._Y = X, y[:, None]
    gp._hyper = dict(kernel_var=s2, lengthscale=l, bias_var=b, noise_var=noise - JITTER)
    with pytest.raises(np.linalg.LinAlgError, match=r'pivot at {}$'.format(j0)):
        gp._fit()
