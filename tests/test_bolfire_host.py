"""BOLFIRE's classifier and constructor without a GPU: the NumPy statement of the device fit
(tests/logreg_double.py) against the reference's scikit-learn fits (tests/golden/
gen_golden_bolfire.py), the optimality rule, and every argument error."""
import numpy as np
import pytest

import logreg_double as L
from bolfire_cases import simple_gaussian_model
from elfi_b200 import ops
from elfi_b200.bo import LCBSC, CostFunction
from elfi_b200.bolfire import BOLFIRE
from elfi_b200.classifier import Classifier, GPClassifier, LogisticRegression
from elfi_b200.samplers import ModelPrior


def cases(g):
    for k in range(int(g['n_cases'])):
        p = 'c{}_'.format(k)
        yield p, g[p + 'X'], g[p + 'y'], float(g[p + 'C']), g[p + 'Xq']


def close(a, b, rel):
    a, b = np.asarray(a), np.asarray(b)
    return np.all(np.abs(a - b) <= rel * (1 + np.abs(b)))


def test_double_matches_tight_liblinear_and_newton(golden):
    g = golden('bolfire_classifier')
    for p, X, y, C, Xq in cases(g):
        f = L.fit(X, y, 'l1', C)
        assert f['converged']
        assert close(L.predict(f, Xq), g[p + 'tight_logratio'], 1e-8), p
        assert close(np.append(f['coef'], f['intercept']),
                     np.append(g[p + 'tight_coef'], g[p + 'tight_intercept']), 1e-6), p
        # at least as optimal as the reference's own fit at its default tolerance
        assert f['objective'] <= g[p + 'default_F'] + 1e-12 * abs(g[p + 'default_F']), p
        f2 = L.fit(X, y, 'l2', C)
        assert close(L.predict(f2, Xq), g[p + 'l2_logratio'], 1e-7), p


def test_optimality_rule_recomputed(golden):
    g = golden('bolfire_classifier')
    for p, X, y, C, _ in cases(g):
        for penalty in ('l1', 'l2'):
            f = L.fit(X, y, penalty, C)
            Xa = L.augmented(X, f['mean'], f['scale'])
            w = np.append(f['coef'], f['intercept'])
            assert L.subgradient_norm(Xa, y, w, penalty, C) <= 1e-10 * C * len(X)


def test_standardisation_rule():
    n = 50
    X = np.column_stack([np.full(n, 0.1), 1e3 + 1e-9 * np.random.RandomState(0).randn(n),
                         np.arange(n, dtype=float)])
    mean, scale = L.standardise(X)
    assert scale[0] == 1.0                      # constant: sklearn's _is_constant_feature
    assert scale[1] != 1.0 and scale[1] < 1e-8  # near-constant but above the rule's bound
    assert scale[2] == np.std(X[:, 2])


def test_config_and_argument_errors():
    assert LogisticRegression().config == {'penalty': 'l1', 'solver': 'liblinear'}
    clf = LogisticRegression({'penalty': 'l2', 'solver': 'liblinear', 'C': 2.0, 'max_iter': 7})
    assert (clf.penalty, clf.C, clf.max_iter) == ('l2', 2.0, 7)
    for key in ('tol', 'fit_intercept', 'class_weight', 'l1_ratio'):
        with pytest.raises(NotImplementedError, match=key):
            LogisticRegression({'penalty': 'l1', 'solver': 'liblinear', key: 1})
    with pytest.raises(NotImplementedError, match='elasticnet'):
        LogisticRegression({'penalty': 'elasticnet'})
    with pytest.raises(NotImplementedError, match='lbfgs'):
        LogisticRegression({'penalty': 'l2', 'solver': 'lbfgs'})
    with pytest.raises(ValueError):
        LogisticRegression({'penalty': 'l1', 'C': 0.0})
    with pytest.raises(TypeError):
        LogisticRegression(class_min='0')
    LogisticRegression(class_min=0.01)
    with pytest.raises(NotImplementedError, match='GPy'):
        GPClassifier()
    with pytest.raises(ValueError, match='2 classes'):
        LogisticRegression().fit(np.zeros((4, 2)), np.ones(4))


def test_ops_argument_errors():
    X = np.random.RandomState(1).randn(6, 3)
    y = np.array([1., -1., 1., -1., 1., -1.])
    with pytest.raises(ValueError, match='penalty'):
        ops.logreg_fit(X, y, penalty='l3')
    with pytest.raises(ValueError, match='C must'):
        ops.logreg_fit(X, y, C=-1.0)
    with pytest.raises(ValueError, match='labels'):
        ops.logreg_fit(X, y * 2)
    with pytest.raises(ValueError, match='both classes'):
        ops.logreg_fit(X, np.ones(6))
    with pytest.raises(ValueError, match='max_iter'):
        ops.logreg_fit(X, y, max_iter=-1)
    with pytest.raises(ValueError, match='LogRegFit'):
        ops.logreg_predict(None, X)


def test_cost_function():
    cost = CostFunction(lambda x: np.sum(x ** 2, axis=1), lambda x: 2 * x, scale=-1)
    x = np.array([[1., 2.], [0., 3.]])
    np.testing.assert_array_equal(cost.evaluate(x), [[-5.], [-9.]])
    np.testing.assert_array_equal(cost.evaluate_gradient(x[0]), [[-2., -4.]])


def test_bolfire_init(cpu_double):
    """The reference's test_bolfire_init on its own toy model."""
    m = simple_gaussian_model(2.6, 4)
    bolfire_method = BOLFIRE(model=m, n_training_data=10)
    assert tuple(bolfire_method.marginal.shape) == (10, 10)
    assert bolfire_method.feature_names == ['power_{}'.format(i) for i in range(10)]
    assert isinstance(bolfire_method.classifier, LogisticRegression)
    assert len(bolfire_method.observed[0]) == 10
    assert isinstance(bolfire_method.prior, ModelPrior)
    assert bolfire_method.bounds is None
    assert bolfire_method.acq_noise_var == 0
    assert bolfire_method.exploration_rate == 10
    assert bolfire_method.update_interval == 1
    assert bolfire_method.n_initial_evidence == 0
    assert isinstance(bolfire_method.acquisition_method, LCBSC)


def test_bolfire_argument_errors(cpu_double):
    m = simple_gaussian_model(2.6, 4)
    with pytest.raises(TypeError, match='marginal'):
        BOLFIRE(m, 10, marginal=[[1.0] * 10])
    with pytest.raises(ValueError, match='Classifier'):
        BOLFIRE(m, 10, classifier='logreg')
    with pytest.raises(ValueError, match='n_initial_evidence'):
        BOLFIRE(m, 10, n_initial_evidence=-1)
    with pytest.raises(TypeError, match='GPyRegression'):
        BOLFIRE(m, 10, target_model=object())
    with pytest.raises(TypeError, match='AcquisitionBase'):
        BOLFIRE(m, 10, acquisition_method=object())
    with pytest.raises(ValueError, match='multiple of batch_size'):
        BOLFIRE(m, 10, batch_size=3)
    b = BOLFIRE(m, 10, bounds={'mu': (-5, 5)})
    with pytest.raises(TypeError, match='positive integer'):
        b.fit(0)
    with pytest.raises(TypeError, match='positive integer'):
        b.fit(2.0)
    assert issubclass(LogisticRegression, Classifier)
