"""NumPy restatement of the logistic-regression entry points of include/elfi_b200.h
(elfi_b200_logreg_fit_f64, elfi_b200_logreg_predict_f64) and their CPU test double -- TEST
INFRASTRUCTURE ONLY.

`standardise` is sklearn's StandardScaler rule (ddof-0 variance with its correction sum, scale 1 for
a constant column by _is_constant_feature).  `fit` solves liblinear's primal with a penalised
intercept to the header's stopping rule: an exact Newton solve for L2, and for L1 proximal Newton
with coordinate descent on the quadratic model.  `objective` and `subgradient_norm` state F and the
optimality measure.  `TABLE` routes both entry points here on top of tests/abi_double.py, so the
unmodified classifier and BOLFIRE host code run without a GPU.
"""
import numpy as np

import abi_double as d

EPS = np.finfo(np.float64).eps
TOL = 1e-10
HEAD = 8
D_MAX = 160


def standardise(X):
    """(mean_, scale_) of StandardScaler over the rows of X."""
    X = np.asarray(X, dtype=np.float64)
    n = X.shape[0]
    mean = X.sum(axis=0) / n
    c = X - mean
    var = (np.sum(c * c, axis=0) - np.sum(c, axis=0) ** 2 / n) / n
    constant = var <= n * EPS * var + (n * mean * EPS) ** 2
    return mean, np.where(constant, 1.0, np.sqrt(var))


def augmented(X, mean, scale):
    Xt = (np.asarray(X, dtype=np.float64) - mean) / scale
    return np.column_stack([Xt, np.ones(len(Xt))])


def _loss(s):
    return np.log1p(np.exp(-np.abs(s))) + np.maximum(-s, 0)


def objective(Xa, y, w, penalty, C):
    """F(w) of the header, on the augmented standardised rows Xa."""
    reg = np.sum(np.abs(w)) if penalty == 'l1' else 0.5 * float(w @ w)
    return reg + C * float(np.sum(_loss(y * (Xa @ w))))


def gradient(Xa, y, w, penalty, C):
    g = Xa.T @ (-C * y / (1 + np.exp(y * (Xa @ w))))
    return g if penalty == 'l1' else g + w


def subgradient(g, w, penalty):
    """The minimum-norm subgradient of F, entry by entry."""
    if penalty == 'l2':
        return np.abs(g)
    return np.where(w > 0, np.abs(g + 1), np.where(w < 0, np.abs(g - 1),
                                                   np.maximum(np.abs(g) - 1, 0)))


def subgradient_norm(Xa, y, w, penalty, C):
    return float(np.max(subgradient(gradient(Xa, y, w, penalty, C), w, penalty)))


def _cd(g, H, w, tol):
    """Coordinate descent on g.delta + delta H delta / 2 + |w + delta|_1."""
    D = len(g)
    dl = np.zeros(D)
    r = g.copy()
    for _ in range(1000):
        for j in range(D):
            z = w[j] + dl[j]
            u = z - r[j] / H[j, j]
            zn = np.sign(u) * max(abs(u) - 1 / H[j, j], 0.0)
            if zn != z:
                r += H[:, j] * (zn - z)
                dl[j] = zn - w[j]
        if np.max(subgradient(r, w + dl, 'l1')) <= tol:
            break
    return dl


def solve(Xa, y, penalty, C, max_iter=100):
    """(w, n_iter, converged) at the header's stopping rule."""
    n, D = Xa.shape
    w = np.zeros(D)
    tol = TOL * C * n
    for it in range(max_iter + 1):
        s = y * (Xa @ w)
        g = gradient(Xa, y, w, penalty, C)
        viol = np.max(subgradient(g, w, penalty))
        if viol <= tol:
            return w, it, True
        if it == max_iter:
            return w, it, False
        e = np.exp(-np.abs(s))
        h = C * e / (1 + e) ** 2
        H = (Xa * h[:, None]).T @ Xa
        if penalty == 'l2':
            dl = -np.linalg.solve(H + np.eye(D), g)
        else:
            dl = _cd(g, H + 1e-12 * np.eye(D), w, max(0.01 * viol, 0.1 * tol))
        F = objective(Xa, y, w, penalty, C)
        pred = float(g @ dl) + (np.sum(np.abs(w + dl)) - np.sum(np.abs(w)) if penalty == 'l1'
                                else 0.0)
        alpha = 1.0
        if not (pred < 0):
            return w, it, False
        if -pred > 1e2 * EPS * F:
            for _ in range(40):
                if objective(Xa, y, w + alpha * dl, penalty, C) - F <= 0.01 * alpha * pred:
                    break
                alpha *= 0.5
            else:
                return w, it, False
        w = w + alpha * dl
    return w, max_iter, False


def fit(X, y, penalty='l1', C=1.0, max_iter=100):
    """dict(mean, scale, coef, intercept, n_iter, converged) of the device's fit."""
    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    mean, scale = standardise(X)
    Xa = augmented(X, mean, scale)
    w, it, conv = solve(Xa, y, penalty, C, max_iter)
    return dict(mean=mean, scale=scale, coef=w[:-1], intercept=w[-1], n_iter=it, converged=conv,
                objective=objective(Xa, y, w, penalty, C))


def predict(f, X, class_min=0.0):
    """The reference's log-likelihood ratio of rows X under the fit f."""
    v = ((np.asarray(X, dtype=np.float64) - f['mean']) / f['scale']) @ f['coef'] + f['intercept']
    with np.errstate(divide='ignore', over='ignore'):
        p = np.maximum(1 / (1 + np.exp(-v)), class_min)
        return np.log(p / (1 - p))


def logreg_fit_f64(ctx, X, ld_row, n, dim, y, penalty, C, max_iter, block, stream):
    d._require(1 <= dim <= D_MAX and 2 <= n and ld_row >= dim, 'logreg_fit: bad shape')
    d._require(penalty in (0, 1) and C > 0 and max_iter >= 0, 'logreg_fit: bad argument')
    Xh = np.array(d._mat(X, n, dim, ld_row))
    yh = np.array(d._vec(y, n))
    out = d._vec(block, HEAD + 3 * dim)
    out[:] = np.nan
    out[5:8] = 0.0
    if not np.all((yh == 1) | (yh == -1)) or np.all(yh == 1) or np.all(yh == -1):
        out[1:3] = 0, -1
        return
    mean, scale = standardise(Xh)
    if not (np.all(np.isfinite(mean)) and np.all(np.isfinite(scale))):
        out[1:3] = 0, -2
        return
    pen = ('l1', 'l2')[penalty]
    Xa = augmented(Xh, mean, scale)
    w, it, conv = solve(Xa, yh, pen, C, max_iter)
    out[:5] = (w[-1], it, 1 if conv else 0, objective(Xa, yh, w, pen, C),
               subgradient_norm(Xa, yh, w, pen, C))
    out[HEAD:] = np.concatenate([mean, scale, w[:-1]])


def logreg_predict_f64(ctx, block, dim, Xq, ld_row, m, class_min, out, stream):
    d._require(1 <= dim <= D_MAX and m >= 0 and ld_row >= dim, 'logreg_predict: bad shape')
    if not m:
        return
    b = np.array(d._vec(block, HEAD + 3 * dim))
    Xh = np.array(d._mat(Xq, m, dim, ld_row))
    f = dict(intercept=b[0], mean=b[HEAD:HEAD + dim], scale=b[HEAD + dim:HEAD + 2 * dim],
             coef=b[HEAD + 2 * dim:])
    v = predict(f, Xh, class_min)
    v[~np.all(np.isfinite(Xh), axis=1) | (b[2] < 0)] = np.nan
    d._vec(out, m)[:] = v


TABLE = {'elfi_b200_logreg_fit_f64': logreg_fit_f64,
         'elfi_b200_logreg_predict_f64': logreg_predict_f64}
