"""Golden fixtures for BOLFIRE, from the UNMODIFIED reference (elfi-dev/elfi, the checkout named by
ELFI_REFERENCE_ROOT) and its scikit-learn classifier.

    ELFI_REFERENCE_ROOT=<checkout> python tests/golden/gen_golden_bolfire.py

* bolfire_classifier.npz -- crafted problems (keys c<k>_*): several d, unequal column scales, a
      constant and a near-constant column, separable data, C in {0.1, 1, 10}.  For each: X, y, C,
      the query rows Xq; the reference LogisticRegression at its default config (coef, intercept,
      log ratios at Xq, and the objective F of include/elfi_b200.h at its weights); the same at
      {'penalty': 'l1', 'solver': 'liblinear', 'tol': 1e-13, 'max_iter': 10**6} ("tight"); and the
      L2 optimum from a NumPy Newton solve to |grad F| <= 1e-12 ("l2").
* bolfire_rounds.npz -- the reference BOLFIRE on arch.get_model(n_obs=100, seed_obs=7) with
      n_training_data = 200, n_initial_evidence = 5, seed = 11, seed_marginal = 3: the marginal
      data, each of the 5 prior-drawn rounds' parameter and value (minus the log ratio, as given to
      the GP), and each round's training data refitted at the tight config.  The GP's update is
      replaced by a recorder (GPy is absent), so no acquisition is reached.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

from ref_shim import import_reference  # noqa: E402

elfi = import_reference()
from elfi.examples import arch  # noqa: E402
from elfi.methods.bo.gpy_regression import GPyRegression  # noqa: E402
from elfi.methods.classifier import LogisticRegression  # noqa: E402

TIGHT = {'penalty': 'l1', 'solver': 'liblinear', 'tol': 1e-13, 'max_iter': 10 ** 6}
ROUNDS = dict(n_training_data=200, n_initial_evidence=5, seed=11, seed_marginal=3, seed_obs=7)


def save(name, **arrays):
    np.savez(os.path.join(HERE, name + '.npz'), **arrays)
    print('wrote', name, len(arrays), 'arrays')


def objective(clf, X, y, C, penalty='l1'):
    """F of the header at a fitted reference classifier's weights."""
    Xs = clf.scaler.transform(X)
    w = np.append(clf.model.coef_[0], clf.model.intercept_[0])
    m = y * (np.column_stack([Xs, np.ones(len(Xs))]) @ w)
    loss = np.sum(np.log1p(np.exp(-np.abs(m))) + np.maximum(-m, 0))
    reg = np.sum(np.abs(w)) if penalty == 'l1' else 0.5 * w @ w
    return reg + C * loss


def newton_l2(X, y, C):
    """The L2 optimum with a penalised intercept, on StandardScaler features."""
    mean = X.mean(axis=0)
    var = X.var(axis=0)
    n = len(X)
    eps = np.finfo(float).eps
    scale = np.where(var <= n * eps * var + (n * mean * eps) ** 2, 1.0, np.sqrt(var))
    Xa = np.column_stack([(X - mean) / scale, np.ones(n)])
    w = np.zeros(Xa.shape[1])
    for _ in range(200):
        m = y * (Xa @ w)
        g = w + Xa.T @ (-C * y / (1 + np.exp(m)))
        if np.max(np.abs(g)) <= 1e-12:
            break
        e = np.exp(-np.abs(m))
        H = np.eye(len(w)) + (Xa * (C * e / (1 + e) ** 2)[:, None]).T @ Xa
        w = w - np.linalg.solve(H, g)
    return w[:-1], w[-1], mean, scale


def case(rs, d, n_per, C, scales=None, shift=0.7, tweak=None):
    X1 = rs.randn(n_per, d) + shift
    X0 = rs.randn(n_per, d) * 1.3
    X = np.vstack([X1, X0])
    if scales is not None:
        X = X * scales
    if tweak is not None:
        tweak(X)
    y = np.concatenate([np.ones(n_per), -np.ones(n_per)])
    Xq = np.vstack([X[:3], X[-2:], X.mean(axis=0, keepdims=True)])
    return X, y, C, Xq


def classifier_cases():
    rs = np.random.RandomState(5)

    def const_cols(X):
        X[:, 1] = 2.5
        X[:, 3] = 1e3 + 1e-9 * rs.randn(len(X))     # near-constant, not constant by the rule

    def separable(X):
        X[: len(X) // 2, 0] += 8.0

    cases = [case(rs, 3, 60, 1.0, scales=np.array([1e-3, 1.0, 1e3])),
             case(rs, 5, 80, 0.1, tweak=const_cols),
             case(rs, 10, 500, 10.0),
             case(rs, 2, 40, 1.0, shift=0.0, tweak=separable),
             case(rs, 17, 200, 1.0, shift=0.2),
             case(rs, 1, 30, 10.0)]
    out = {}
    for k, (X, y, C, Xq) in enumerate(cases):
        p = 'c{}_'.format(k)
        out.update({p + 'X': X, p + 'y': y, p + 'C': np.float64(C), p + 'Xq': Xq})
        for name, cfg in (('default', {'penalty': 'l1', 'solver': 'liblinear', 'C': C}),
                          ('tight', dict(TIGHT, C=C))):
            clf = LogisticRegression(cfg)
            clf.fit(X, y)
            out[p + name + '_coef'] = clf.model.coef_[0]
            out[p + name + '_intercept'] = np.float64(clf.model.intercept_[0])
            out[p + name + '_logratio'] = clf.predict_log_likelihood_ratio(Xq)
            out[p + name + '_F'] = np.float64(objective(clf, X, y, C))
            out[p + name + '_n_iter'] = np.int64(clf.model.n_iter_[0])
        coef, b, mean, scale = newton_l2(X, y, C)
        v = ((Xq - mean) / scale) @ coef + b
        p1 = 1 / (1 + np.exp(-v))
        out[p + 'l2_coef'], out[p + 'l2_intercept'] = coef, np.float64(b)
        out[p + 'l2_logratio'] = np.log(p1 / (1 - p1))
    out['n_cases'] = np.int64(len(cases))
    return out


class RecordingGP(GPyRegression):
    """The reference GP with its update replaced by a recorder (GPy is absent)."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.records = []

    @property
    def n_evidence(self):
        return len(self.records)

    def update(self, x, y, optimize=False):
        self.records.append((np.array(x, dtype=float).reshape(-1), np.array(y).reshape(-1),
                             bool(optimize)))


def rounds():
    m = arch.get_model(n_obs=100, seed_obs=ROUNDS['seed_obs'])
    bounds = {'t1': (-1, 1), 't2': (0, 1)}
    gp = RecordingGP(m.parameter_names, bounds)
    seen = []
    bolfire = elfi.BOLFIRE(m, ROUNDS['n_training_data'], seed_marginal=ROUNDS['seed_marginal'],
                           bounds=bounds, n_initial_evidence=ROUNDS['n_initial_evidence'],
                           target_model=gp, seed=ROUNDS['seed'])
    fit = bolfire.predict_log_ratio

    def spy(X, y, X_obs):
        seen.append(np.array(X))
        return fit(X, y, X_obs)
    bolfire.predict_log_ratio = spy
    bolfire.fit(ROUNDS['n_initial_evidence'], bar=False)
    theta = np.array([r[0] for r in gp.records])
    value = np.array([r[1][0] for r in gp.records])
    y = np.concatenate([np.ones(ROUNDS['n_training_data']), -np.ones(ROUNDS['n_training_data'])])
    tight = []
    for X in seen:
        clf = LogisticRegression(TIGHT)
        clf.fit(X, y)
        tight.append(-clf.predict_log_likelihood_ratio(bolfire.observed)[0])
    return dict(marginal=np.array(bolfire.marginal), theta=theta, value=value,
                value_tight=np.array(tight), observed=np.array(bolfire.observed),
                optimize=np.array([r[2] for r in gp.records]),
                n_iter=np.array([a['parameters']['n_iter'][0]
                                 for a in bolfire.classifier_attributes]),
                **{k: np.int64(v) for k, v in ROUNDS.items()})


if __name__ == '__main__':
    save('bolfire_classifier', **classifier_cases())
    save('bolfire_rounds', **rounds())
