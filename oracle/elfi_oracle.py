"""CPU oracle for the ELFI sampler / BOLFI hot path.

TEST INFRASTRUCTURE ONLY -- not part of the product.  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference``
legs may import this module.  ``elfi_b200`` never does: the product path has no CPU
fallback and fails loudly when the CUDA library is missing.

Each function restates one reference function (paths relative to the root of elfi-dev/elfi) and
is pinned against (i) the reference itself, imported with oracle/ref_shim.py when the
golden fixtures under tests/golden/ were generated, and (ii) the installed SciPy/NumPy
that the reference calls (tests/test_oracle.py).

Parity status: sampler path (distance, summaries, merge, quantile, weights) PINNED by
golden fixtures generated from the reference.  GP posterior PINNED against the reference's
own NumPy restatement (gpy_regression.py:127-160, 206-218) and scikit-learn.  GP
hyper-parameter optimisation: PARITY UNPINNED (GPy absent; see DESIGN.md).
"""
import ctypes
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        path = os.path.join(_HERE, 'libelfi_oracle.so')
        if not os.path.exists(path):
            import subprocess
            subprocess.check_call(['make', '-C', _HERE, '-s'])
        _LIB = ctypes.CDLL(path)
        _LIB.oracle_pairwise_sum.restype = ctypes.c_double
        _LIB.oracle_accept.restype = ctypes.c_int64
    return _LIB


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def _c64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _row_chunks(B, threads):
    threads = max(1, min(int(threads), B if B > 0 else 1))
    edges = np.linspace(0, B, threads + 1).astype(np.int64)
    return [(int(edges[i]), int(edges[i + 1])) for i in range(threads) if edges[i + 1] > edges[i]]


def _parallel_rows(fn, B, threads):
    chunks = _row_chunks(B, threads)
    if len(chunks) <= 1:
        for lo, hi in chunks:
            fn(lo, hi)
        return
    with ThreadPoolExecutor(len(chunks)) as ex:
        list(ex.map(lambda c: fn(*c), chunks))


# ----------------------------------------------------------------------------- distance
def cdist_euclid(S, obs, w=None, threads=1):
    """scipy.spatial.distance.cdist(S, obs(1,D), 'euclidean', w=w) flattened to (B,).

    Reference: elfi/model/utils.py:37-52 calling elfi/model/elfi_model.py:1037 / :1131.
    Sequential left-to-right fp64 accumulation, no FMA (oracle/c/elfi_oracle.c).
    """
    S = _c64(S)
    if S.ndim == 1:
        S = S[:, None]
    obs = _c64(obs).reshape(-1)
    B, D = S.shape
    assert obs.shape[0] == D
    wv = None if w is None else _c64(w).reshape(-1)
    out = np.empty(B, dtype=np.float64)
    lib = _lib()

    def run(lo, hi):
        lib.oracle_cdist_euclid(_p(S[lo:hi]), ctypes.c_int64(S.shape[1]), ctypes.c_int64(hi - lo),
                                ctypes.c_int64(D), _p(obs), _p(wv), _p(out[lo:hi]))
    _parallel_rows(run, B, threads)
    return out


METRIC_CODES = {'sqeuclidean': 1, 'cityblock': 2, 'chebyshev': 3, 'minkowski': 4}


def cdist_metric(S, obs, metric, p=2.0):
    """scipy.spatial.distance.cdist(S, obs(1,D), metric[, p=p]) flattened to (B,) for the other
    metrics elfi.Distance accepts (elfi/model/elfi_model.py:1016-1037), sequential fp64."""
    S = _c64(S)
    if S.ndim == 1:
        S = S[:, None]
    obs = _c64(obs).reshape(-1)
    out = np.empty(len(S), dtype=np.float64)
    _lib().oracle_cdist_metric(_p(S), ctypes.c_int64(S.shape[1]), ctypes.c_int64(len(S)),
                               ctypes.c_int64(S.shape[1]), _p(obs),
                               ctypes.c_int32(METRIC_CODES[metric]), ctypes.c_double(p), _p(out))
    return out


def cdist_seuclidean(S, obs, V):
    """scipy.spatial.distance.cdist(S, obs(1,D), 'seuclidean', V=V) flattened to (B,): the
    Distance('seuclidean', ..., V=) node of elfi/model/elfi_model.py:1016-1037, in the two-sum
    order of SciPy's compiled loop (oracle/c/elfi_oracle.c)."""
    S = _c64(S)
    if S.ndim == 1:
        S = S[:, None]
    obs = _c64(obs).reshape(-1)
    V = _c64(V).reshape(-1)
    assert obs.shape[0] == S.shape[1] == V.shape[0]
    out = np.empty(len(S), dtype=np.float64)
    _lib().oracle_cdist_seuclidean(_p(S), ctypes.c_int64(S.shape[1]), ctypes.c_int64(len(S)),
                                   ctypes.c_int64(S.shape[1]), _p(obs), _p(V), _p(out))
    return out


def nested_distance(S, obs, weights, threads=1):
    """AdaptiveDistance.nested_distance (elfi/model/elfi_model.py:1135-1151).

    ``weights`` is the list state['w']: entry None => unweighted cdist, else cdist(w=wk**2).
    Returns (B, K).
    """
    S = _c64(S)
    obs = _c64(obs).reshape(-1)
    B, D = S.shape
    K = len(weights)
    W = np.zeros((K, D))
    unweighted = np.zeros(K, dtype=np.int32)
    for k, wk in enumerate(weights):
        if wk is None:
            unweighted[k] = 1
        else:
            W[k] = np.asarray(wk, dtype=np.float64) ** 2
    out = np.empty((B, K))
    lib = _lib()

    def run(lo, hi):
        lib.oracle_nested_distance(_p(S[lo:hi]), ctypes.c_int64(D), ctypes.c_int64(hi - lo),
                                   ctypes.c_int64(D), _p(obs), _p(W), _p(unweighted),
                                   ctypes.c_int64(K), _p(out[lo:hi]))
    _parallel_rows(run, B, threads)
    return out


def accept_indices(d, thresholds):
    """Rows with all_k(d[:,k] <= thr[k]) (elfi/methods/inference/samplers.py:223-225)."""
    d = _c64(d)
    d2 = d.reshape(len(d), -1)
    thr = _c64(np.atleast_1d(thresholds))
    idx = np.empty(len(d2), dtype=np.int32)
    n = _lib().oracle_accept(_p(d2), ctypes.c_int64(d2.shape[0]), ctypes.c_int64(d2.shape[1]),
                             _p(thr), _p(idx))
    return idx[:n].copy()


# ---------------------------------------------------------------------------- summaries
def pairwise_sum(a):
    """NumPy's pairwise float64 summation order (DOUBLE_pairwise_sum)."""
    a = _c64(a).reshape(-1)
    return float(_lib().oracle_pairwise_sum(_p(a), ctypes.c_int64(a.size)))


def autocov(x, lag=1, threads=1):
    """elfi/examples/ma2.py:40-59."""
    x = _c64(np.atleast_2d(x))
    B, n = x.shape
    out = np.empty(B)
    lib = _lib()

    def run(lo, hi):
        lib.oracle_autocov(_p(x[lo:hi]), ctypes.c_int64(n), ctypes.c_int64(hi - lo),
                           ctypes.c_int64(n), ctypes.c_int64(lag), _p(out[lo:hi]))
    _parallel_rows(run, B, threads)
    return out


def meanvar(y, threads=1):
    """ss_mean, ss_var of elfi/examples/gauss.py:142-173 (np.mean / np.var over axis 1)."""
    y = _c64(y)
    B, n = y.shape
    mean = np.empty(B)
    var = np.empty(B)
    lib = _lib()

    def run(lo, hi):
        lib.oracle_meanvar(_p(y[lo:hi]), ctypes.c_int64(n), ctypes.c_int64(hi - lo),
                           ctypes.c_int64(n), _p(mean[lo:hi]), _p(var[lo:hi]))
    _parallel_rows(run, B, threads)
    return mean, var


# ------------------------------------------------------------- adaptive-distance moments
def welford_add(store, data):
    """AdaptiveDistance.add_data (elfi/model/elfi_model.py:1104-1125).

    store = [n, mean, M2]; returns the new store and scale = sqrt(M2 / n)."""
    data = _c64(data)
    if data.ndim == 1:
        data = data[:, None]
    n0, m0, s0 = store
    n1 = n0 + len(data)
    delta_1 = data - m0
    m1 = m0 + np.sum(delta_1, axis=0) / n1
    delta_2 = data - m1
    s1 = s0 + np.sum(delta_1 * delta_2, axis=0)
    return [n1, m1, s1], np.sqrt(s1 / n1)


# ------------------------------------------------------------------ rejection bookkeeping
def merge_batch(samples, batch, n_samples, threshold, discrepancy_name):
    """Rejection._merge_batch (elfi/methods/inference/samplers.py:209-237), in place.

    ``samples``: dict name -> (n_samples + B, ...) buffers, distances initialised to +inf.
    Sort key = last distance column; np.argsort (unstable kind, ties have measure zero).
    """
    d = batch[discrepancy_name]
    if threshold is None:
        accepted = slice(None, None)
        num_accepted = len(d)
    else:
        accepted = d <= threshold
        accepted = np.all(np.atleast_2d(np.transpose(accepted)), axis=0)
        num_accepted = int(np.sum(accepted))
    if num_accepted > 0:
        for node, v in samples.items():
            v[-num_accepted:] = batch[node][accepted]
    sort_distance = np.atleast_2d(np.transpose(samples[discrepancy_name]))[-1]
    sort_mask = np.argsort(sort_distance)
    for k, v in samples.items():
        v[:] = v[sort_mask]
    return num_accepted


def topn_smallest(d, n):
    """Indices of the n smallest entries of d, ascending by value (ties by index)."""
    order = np.argsort(d, kind='stable')
    return order[:n]


# ----------------------------------------------------------------------- SMC utilities
def weighted_sample_quantile(x, alpha, weights=None):
    """elfi/methods/utils.py:379-411."""
    x = np.asarray(x)
    index = np.argsort(x)
    if alpha == 0:
        return x[index[0]]
    if weights is None:
        weights = np.ones(len(index))
    weights = weights / np.sum(weights)
    sorted_weights = weights[index]
    cum_weights = np.insert(np.cumsum(sorted_weights), 0, 0)
    cum_weights[-1] = 1.0
    index_alpha = np.where(np.logical_and(cum_weights[:-1] < alpha,
                                          alpha <= cum_weights[1:]))[0][0]
    return x[index][index_alpha]


def weighted_var(x, weights=None):
    """elfi/methods/utils.py:108-139."""
    x = np.asarray(x, dtype=np.float64)
    if weights is None:
        weights = np.ones(len(x))
    V_1 = np.sum(weights)
    V_2 = np.sum(weights ** 2)
    xbar = np.average(x, weights=weights, axis=0)
    numerator = weights.dot((x - xbar) ** 2)
    return numerator / (V_1 - (V_2 / V_1))


def gm_logpdf(x, means, cov, weights=None, block=4096):
    """GMDistribution.logpdf (elfi/methods/utils.py:146-197).

    log sum_j w_j N(x_i; m_j, cov) with w normalised; SciPy's multivariate_normal.pdf
    for a shared covariance is exp(-0.5*(k*log(2*pi) + logdet + maha)).  The reference
    sums plain densities (no log-sum-exp), so underflow to -inf is reproduced.
    Tolerance-level parity (1e-5 relative on the resulting weights)."""
    x = np.atleast_2d(_c64(x))
    means = np.atleast_2d(_c64(means))
    N, p = means.shape
    if x.shape[1] != p:
        x = x.reshape(-1, p)
    cov = np.atleast_2d(_c64(cov))
    if cov.shape == (1, 1) and p > 1:
        cov = np.eye(p) * cov[0, 0]
    if weights is None:
        weights = np.ones(N)
    w = _c64(weights)
    w = w / np.sum(w)
    prec = np.linalg.inv(cov)
    _, logdet = np.linalg.slogdet(cov)
    lognorm = -0.5 * (p * np.log(2 * np.pi) + logdet)
    out = np.zeros(len(x))
    for lo in range(0, N, block):
        m = means[lo:lo + block]
        diff = x[:, None, :] - m[None, :, :]
        maha = np.einsum('ijk,kl,ijl->ij', diff, prec, diff)
        out += np.exp(lognorm - 0.5 * maha) @ w[lo:lo + block]
    with np.errstate(divide='ignore'):
        return np.log(out)


def smc_weights_and_cov(params, prior_logpdf, prev_means, prev_cov, prev_weights):
    """SMC._compute_weights_means_and_cov (elfi/methods/inference/samplers.py:508-534)."""
    params = np.atleast_2d(_c64(params))
    if prev_means is None:
        w = np.ones(len(params))
    else:
        q = gm_logpdf(params, prev_means, prev_cov, prev_weights)
        w = np.exp(prior_logpdf - q)
    if np.count_nonzero(w) == 0:
        raise RuntimeError("All sample weights are zero.")
    cov = 2 * np.diag(weighted_var(params, w))
    if not np.all(np.isfinite(cov)):
        cov = np.diag(np.ones(params.shape[1]))
    return w, cov


# -------------------------------------------------------------------------------- GP
def gp_gram(X, kernel_var, lengthscale, bias_var):
    """K = s2 * exp(-r2 / (2 l^2)) + b, restating gpy_regression.py:132-133 (RBF+Bias)."""
    X = np.atleast_2d(_c64(X))
    x2 = np.sum(X ** 2., 1)
    r2 = x2[:, None] + x2[None, :] - 2. * X.dot(X.T)
    r2 = np.maximum(r2, 0.0)
    return kernel_var * np.exp(r2 * (-0.5 / lengthscale ** 2)) + bias_var


def gp_fit(X, Y, kernel_var, lengthscale, bias_var, noise_var, jitter=1e-8):
    """Posterior factors GPy exposes and gpy_regression.py:152-158 caches:
    L = chol(K + (noise+jitter) I)  (woodbury_chol), alpha = Ky^-1 y (woodbury_vector)."""
    import scipy.linalg as sl
    K = gp_gram(X, kernel_var, lengthscale, bias_var)
    Ky = K + (noise_var + jitter) * np.eye(len(K))
    L = sl.cholesky(Ky, lower=True)
    alpha = sl.cho_solve((L, True), _c64(Y).reshape(-1, 1))
    return L, alpha


def gp_predict(x, X, L, alpha, kernel_var, lengthscale, bias_var, noise_var=None):
    """GP mean/var at rows of x; diagonal form of gpy_regression.py:132-138
    (the reference's cached-RBF path returns the full (m,m) matrix for m>1; the diagonal
    is what GPy's predict returns and what LCBSC consumes, acquisition.py:276-280)."""
    import scipy.linalg as sl
    x = np.atleast_2d(_c64(x))
    X = np.atleast_2d(_c64(X))
    r2 = np.sum(x ** 2., 1)[:, None] + np.sum(X ** 2., 1)[None, :] - 2. * x.dot(X.T)
    r2 = np.maximum(r2, 0.0)
    kx = kernel_var * np.exp(r2 * (-0.5 / lengthscale ** 2)) + bias_var
    mu = kx.dot(alpha)
    v = sl.solve_triangular(L, kx.T, lower=True)
    var = (kernel_var + bias_var) - np.sum(v * v, axis=0)[:, None]
    if noise_var is not None:
        var = var + noise_var
    return mu, var


def gp_predictive_gradients(x, X, L, alpha, kernel_var, lengthscale, bias_var):
    """gpy_regression.py:206-218 for each query row (returns (m,p), (m,p))."""
    import scipy.linalg as sl
    x = np.atleast_2d(_c64(x))
    X = np.atleast_2d(_c64(X))
    factor = -0.5 / lengthscale ** 2
    gm = np.empty_like(x)
    gv = np.empty_like(x)
    for i in range(len(x)):
        xi = x[i:i + 1]
        r2 = np.sum(xi ** 2., 1)[:, None] + np.sum(X ** 2., 1)[None, :] - 2. * xi.dot(X.T)
        kx = kernel_var * np.exp(r2 * factor)
        dkdx = 2. * factor * (xi - X) * kx.T
        gm[i] = dkdx.T.dot(alpha).T
        v = sl.solve_triangular(L, kx.T + bias_var, lower=True)
        dvdx = sl.solve_triangular(L, dkdx, lower=True)
        gv[i] = (-2. * dvdx.T.dot(v).T)
    return gm, gv


def lcbsc_beta(t, input_dim, exploration_rate=10):
    """LCBSC._beta (elfi/methods/bo/acquisition.py:256-260)."""
    t = t + 1
    delta = 1 / exploration_rate
    return 2 * np.log(t ** (2 * input_dim + 2) * np.pi ** 2 / (3 * delta))


def lcbsc(mean, var, beta):
    """LCBSC.evaluate (elfi/methods/bo/acquisition.py:276-280)."""
    return mean - np.sqrt(beta * var)


def lcbsc_gradient(var, grad_mean, grad_var, beta):
    """LCBSC.evaluate_gradient (elfi/methods/bo/acquisition.py:296-301)."""
    return grad_mean - 0.5 * grad_var * np.sqrt(beta / var)


# ------------------------------------------------------------------------------ KLIEP
def kliep_fit(x, y, weights_x=None, weights_y=None, sigma=1.0, n=100, epsilon=0.001, max_iter=200,
              abs_tol=0.01, conv_check_interval=20):
    """Vectorised restatement of DensityRatioEstimation.fit / _KLIEP / max_ratio
    (elfi/methods/density_ratio_estimation.py:71-207).  Returns (alpha, max_ratio)."""
    x = _c64(x).reshape(len(x), -1)
    y = _c64(y).reshape(len(y), -1)
    theta = x[:n]
    wx = np.ones(len(x)) if weights_x is None else _c64(weights_x)
    wy = np.ones(len(y)) if weights_y is None else _c64(weights_y)
    wy_n = wy / np.sum(wy)

    def basis(a, c):
        d2 = ((a[:, None, :] - c[None, :, :]) ** 2).sum(-1)
        return np.exp(-0.5 * d2 / sigma / sigma)
    A = basis(x, theta)
    b = basis(theta, y) @ wy_n
    b_normalized = b / np.dot(b, b)
    alpha = 1 / n * np.ones(n)
    target_prev = A @ alpha
    non_null = np.any(A > 1e-64, axis=1)
    A_full, w_full = A[non_null], wx[non_null]
    for i in range(max_iter):
        dA = A_full.T @ (w_full / (A_full @ alpha))
        alpha = alpha + epsilon * dA
        alpha = np.maximum(0, alpha + (1 - np.dot(b, alpha)) * b_normalized)
        alpha = alpha / np.dot(b, alpha)
        if i % conv_check_interval == 0:
            target = A @ alpha
            if np.linalg.norm(target - target_prev) < abs_tol:
                break
            target_prev = target
    return alpha, float(np.max(A @ alpha))
