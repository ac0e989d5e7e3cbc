"""NumPy restatement of the synthetic likelihood of include/elfi_b200.h (elfi_b200_synlik_f64) and
its CPU test double -- TEST INFRASTRUCTURE ONLY.

`synlik` states the device's definition with NumPy and SciPy: np.cov moments, whitening as
W Sigma W^T and W (y - mu), Warton shrinkage (1 - l) Sigma + l diag(Sigma_jj + 1e-5), one Cholesky
factor, and -inf for a group with a non-finite input or a pivot L_jj^2 <= 1e6 eps max_i Sigma_ii.
`TABLE` routes the entry point here on top of tests/abi_double.py (through
`abi_double.install`), so the unmodified BSL host code runs without a GPU.
"""
import numpy as np
import scipy.linalg
from scipy.special import gammaln

import abi_double as d

PIVOT_CUT = 1e6 * np.finfo(np.float64).eps
D_MAX = 160


def log_c(k, nu):
    """log c(k, nu) of Ghurye and Olkin (1969)."""
    return (-k * nu / 2 * np.log(2) - k * (k - 1) / 4 * np.log(np.pi)
            - np.sum(gammaln(0.5 * (nu - np.arange(k)))))


def _gaussian(sig, b, estimator, n):
    dim = len(b)
    try:
        L = np.linalg.cholesky(sig)
    except np.linalg.LinAlgError:
        return -np.inf
    piv = np.diag(L) ** 2
    if not np.all(np.isfinite(piv)) or np.any(piv <= PIVOT_CUT * np.max(np.diag(sig))):
        return -np.inf
    z = scipy.linalg.solve_triangular(L, b, lower=True)
    logdet = 2 * np.sum(np.log(np.diag(L)))
    m = float(z @ z)
    if estimator == 'standard':
        return -0.5 * (dim * np.log(2 * np.pi) + logdet + m)
    with np.errstate(divide='ignore'):
        logdet_psi = dim * np.log(n - 1) + logdet + np.log(abs(1 - n * m / (n - 1) ** 2))
    a = log_c(dim, n - 2) - log_c(dim, n - 1) - 0.5 * dim * np.log(1 - 1 / n)
    return (-0.5 * dim * np.log(2 * np.pi) + a - 0.5 * (n - dim - 2) * (np.log(n - 1) + logdet)
            + 0.5 * (n - dim - 3) * logdet_psi)


def synlik(S, y, estimator='standard', penalties=None, W=None):
    """ll (G,) of S (G, n, d) or (n, d), or (G, K) for K penalties."""
    S = np.asarray(S, dtype=np.float64)
    if S.ndim == 2:
        S = S[None]
    G, n, _ = S.shape
    y = np.asarray(y, dtype=np.float64).reshape(-1)
    pens = [None] if penalties is None else list(np.asarray(penalties, dtype=float).reshape(-1))
    out = np.empty((G, len(pens)))
    for g in range(G):
        X = S[g]
        if not np.all(np.isfinite(X)):
            out[g] = -np.inf
            continue
        mu = X.mean(axis=0)
        sig = np.atleast_2d(np.cov(X, rowvar=False))
        b = y - mu
        if W is not None:
            sig = W @ sig @ W.T
            b = W @ b
        for k, lam in enumerate(pens):
            s = sig if lam is None else (1 - lam) * sig + lam * np.diag(np.diag(sig) + 1e-5)
            out[g, k] = _gaussian(s, b, estimator, n)
    return out[:, 0] if penalties is None else out


def synlik_f64(ctx, S, ld_row, ld_group, G, n, dim, y, W, estimator, penalties_host, K, loglik,
               stream):
    d._require(1 <= dim <= D_MAX and n >= 2 and G >= 0 and ld_row >= dim and ld_group >= 0,
               'synlik: bad shape')
    d._require(estimator in (0, 1), 'synlik: bad estimator')
    d._require(estimator == 0 or (not d._addr(W) and K == 0),
               'synlik: whitening and penalties apply to the standard estimator only')
    pens = None
    if K:
        pens = np.array(d._vec(penalties_host, K))
        d._require(np.all((pens >= 0) & (pens <= 1)), 'synlik: penalty outside [0, 1]')
    if not G:
        return
    span = (G - 1) * ld_group + (n - 1) * ld_row + dim
    X = np.array(np.lib.stride_tricks.as_strided(d._vec(S, span), (G, n, dim),
                                                 (8 * ld_group, 8 * ld_row, 8)))
    Wm = np.array(d._mat(W, dim, dim)) if d._addr(W) else None
    ll = synlik(X, np.array(d._vec(y, dim)), ('standard', 'unbiased')[estimator], pens, Wm)
    d._vec(loglik, G * max(K, 1))[:] = ll.reshape(-1)


TABLE = {'elfi_b200_synlik_f64': synlik_f64}
