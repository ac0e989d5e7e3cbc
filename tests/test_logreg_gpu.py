"""The device logistic regression (elfi_b200_logreg_fit_f64 / _predict_f64) against its NumPy
statement (tests/logreg_double.py) and the reference's scikit-learn fits (the committed
tests/golden/bolfire_classifier.npz)."""
import numpy as np
import pytest
import torch

import logreg_double as L
from elfi_b200 import ops
from elfi_b200.classifier import LogisticRegression

pytestmark = pytest.mark.gpu


def problem(d, n_per, seed):
    rs = np.random.RandomState(seed)
    scales = np.exp(rs.uniform(-2, 2, d))
    X = np.vstack([rs.randn(n_per, d) + 0.3, rs.randn(n_per, d) * 1.3]) * scales
    y = np.r_[np.ones(n_per), -np.ones(n_per)]
    return X, y


def device_fit(X, y, penalty, C):
    f = ops.logreg_fit(torch.as_tensor(X, device='cuda'), y, penalty=penalty, C=C)
    f.check()
    return f


def weights(f):
    return np.append(f.coef_, f.intercept_)


def optimality(f, X, y, penalty, C):
    Xa = L.augmented(X, f.mean_, f.scale_)
    w = weights(f)
    return L.subgradient_norm(Xa, y, w, penalty, C), L.objective(Xa, y, w, penalty, C)


@pytest.mark.parametrize('d', [1, 2, 17, 32, 33, 64, 160])
@pytest.mark.parametrize('n_per', ['d+1', 500, 20000])
@pytest.mark.parametrize('penalty', ['l1', 'l2'])
def test_device_matches_double(d, n_per, penalty):
    n_per = d + 1 if n_per == 'd+1' else n_per
    X, y = problem(d, n_per, seed=d * 7 + n_per)
    Xq = X[::max(1, len(X) // 7)]
    for C in (0.1, 1.0, 10.0):
        f = device_fit(X, y, penalty, C)
        assert f.converged, (d, n_per, penalty, C, f.n_iter)
        ref = L.fit(X, y, penalty, C)
        np.testing.assert_allclose(f.mean_, ref['mean'], rtol=1e-12, atol=1e-12 * np.abs(X).max())
        np.testing.assert_allclose(f.scale_, ref['scale'], rtol=1e-10)
        viol, F = optimality(f, X, y, penalty, C)
        assert viol <= 2e-10 * C * len(X)
        assert abs(F - ref['objective']) <= 1e-9 * (1 + abs(ref['objective']))
        assert abs(f.objective - F) <= 1e-9 * (1 + abs(F))
        v = ops.logreg_predict(f, Xq).cpu().numpy()
        vr = L.predict(ref, Xq)
        if penalty == 'l2' or n_per >= 500:      # the L1 optimum of a separable set need not be unique
            assert np.all(np.abs(v - vr) <= 1e-6 * (1 + np.abs(vr))), (d, n_per, penalty, C)


def test_golden_cases():
    g = np.load(__import__('os').path.join(__import__('os').path.dirname(__file__), 'golden',
                                           'bolfire_classifier.npz'))
    for k in range(int(g['n_cases'])):
        p = 'c{}_'.format(k)
        X, y, C, Xq = g[p + 'X'], g[p + 'y'], float(g[p + 'C']), g[p + 'Xq']
        f = device_fit(X, y, 'l1', C)
        assert f.converged
        v = ops.logreg_predict(f, Xq).cpu().numpy()
        ref = g[p + 'tight_logratio']
        assert np.all(np.abs(v - ref) <= 1e-8 * (1 + np.abs(ref))), p
        viol, F = optimality(f, X, y, 'l1', C)
        assert viol <= 2e-10 * C * len(X)
        assert F <= g[p + 'default_F'], p      # at least as optimal as the reference's own fit
        f2 = device_fit(X, y, 'l2', C)
        v2 = ops.logreg_predict(f2, Xq).cpu().numpy()
        # the L2 optimum on the device's own standardisation; against the golden's NumPy means,
        # a near-constant column (case 1: scale 1e-9 around 1e3) moves x~ by the last bits of its
        # mean divided by its scale, about 1e-4, so that comparison is loose
        w, _, _ = L.solve(L.augmented(X, f2.mean_, f2.scale_), y, 'l2', C)
        own = L.predict(dict(mean=f2.mean_, scale=f2.scale_, coef=w[:-1], intercept=w[-1]), Xq)
        assert np.all(np.abs(v2 - own) <= 1e-8 * (1 + np.abs(own))), p
        assert np.all(np.abs(v2 - g[p + 'l2_logratio']) <= 1e-4 * (1 + np.abs(v2))), p


def test_constant_columns_strides_and_repeat():
    rs = np.random.RandomState(3)
    n = 400
    X = rs.randn(n, 6)
    X[:, 1] = 0.1                                      # constant: scale 1
    X[:, 3] = 1e3 + 1e-9 * rs.randn(n)                 # near-constant, above the rule's bound
    y = np.r_[np.ones(n // 2), -np.ones(n // 2)]
    X[: n // 2, 0] += 1.0
    f = device_fit(X, y, 'l1', 1.0)
    mean, scale = L.standardise(X)
    assert f.scale_[1] == 1.0 and scale[1] == 1.0
    assert f.scale_[3] != 1.0 and abs(f.scale_[3] / scale[3] - 1) < 1e-6
    big = torch.zeros((n, 11), dtype=torch.float64, device='cuda')
    big[:, :6] = torch.as_tensor(X, device='cuda')
    strided = ops.logreg_fit(big[:, :6], y, penalty='l1', C=1.0)
    assert torch.equal(strided.block, f.block)
    again = ops.logreg_fit(torch.as_tensor(X, device='cuda'), y, penalty='l1', C=1.0)
    assert torch.equal(again.block, f.block)
    p1 = ops.logreg_predict(f, big[:5, :6])
    assert torch.equal(p1, ops.logreg_predict(f, X[:5]))


def test_failures_raise():
    X, y = problem(4, 50, 1)
    bad = X.copy()
    bad[7, 2] = np.nan
    clf = LogisticRegression()
    with pytest.raises(ValueError):
        clf.fit(bad, y)
    clf.fit(X, y)
    with pytest.raises(ValueError):
        clf.predict_log_likelihood_ratio(bad[:10])
    f = ops.logreg_fit(torch.as_tensor(X, device='cuda'),
                       torch.as_tensor(y * 0.5, device='cuda'))
    with pytest.raises(ValueError, match='labels'):
        f.check()
    assert np.isnan(ops.logreg_predict(f, X[:2]).cpu().numpy()).all()
    ones = torch.ones(len(X), dtype=torch.float64, device='cuda')
    with pytest.raises(ValueError, match='labels'):
        ops.logreg_fit(X, ones).check()


def test_classifier_attributes_and_class_min():
    X, y = problem(5, 100, 2)
    clf = LogisticRegression(class_min=0.3)
    clf.fit(X, np.where(y > 0, 2, 0))                 # the larger label is the positive class
    a = clf.attributes['parameters']
    assert np.shape(a['coef_']) == (1, 5) and len(a['intercept_']) == 1 and a['n_iter'][0] > 0
    v = clf.predict_log_likelihood_ratio(X[-20:])
    assert np.all(v >= np.log(0.3 / 0.7) - 1e-12)
