"""BOLFIRE's host logic under the CPU double of the C ABI: the host ARCH model reproduces the
reference's marginal data and prior-drawn rounds (tests/golden/gen_golden_bolfire.py), and each
round's value is the optimum of its classifier."""
import numpy as np

import abi_double
import logreg_double
from elfi_b200.bolfire import BOLFIRE
from elfi_b200.examples import arch


def run(g):
    m = arch.get_model(n_obs=100, seed_obs=int(g['seed_obs']))
    bounds = {'t1': (-1, 1), 't2': (0, 1)}
    bolfire = BOLFIRE(m, int(g['n_training_data']), seed_marginal=int(g['seed_marginal']),
                      bounds=bounds, n_initial_evidence=int(g['n_initial_evidence']),
                      seed=int(g['seed']))
    post = bolfire.fit(int(g['n_initial_evidence']), bar=False)
    return bolfire, post


def test_rounds_match_reference(cpu_double, monkeypatch, golden):
    abi_double.install(monkeypatch, logreg_double.TABLE)
    g = golden('bolfire_rounds')
    bolfire, post = run(g)
    np.testing.assert_array_equal(bolfire.observed, g['observed'])
    np.testing.assert_array_equal(bolfire.marginal.cpu().numpy(), g["marginal"])
    gp = bolfire.target_model
    np.testing.assert_array_equal(gp.X, g['theta'])
    v, ref = gp.Y[:, 0], g['value_tight']
    assert np.all(np.abs(v - ref) <= 1e-7 * (1 + np.abs(ref)))
    # one fit and one predict per round
    n = int(g['n_initial_evidence'])
    assert cpu_double.CALLS.count('elfi_b200_logreg_fit_f64') == n
    assert cpu_double.CALLS.count('elfi_b200_logreg_predict_f64') == n
    attrs = post.classifier_attributes
    assert len(attrs) == n
    for a in attrs:
        p = a['parameters']
        assert np.shape(p['coef_']) == (1, 17)
        assert np.shape(p['intercept_']) == (1,) and np.shape(p['n_iter']) == (1,)
    assert bolfire.n_evidence == n and bolfire.state['n_sim'] == n * int(g['n_training_data'])


def test_host_classifier(cpu_double, monkeypatch, golden):
    """A user Classifier gets NumPy (X, y) of the round's simulations then the marginal data."""
    abi_double.install(monkeypatch, logreg_double.TABLE)
    g = golden('bolfire_rounds')
    seen = []

    from elfi_b200.classifier import Classifier

    class Host(Classifier):
        def __init__(self):
            self.f = None

        def fit(self, X, y):
            seen.append((type(X), X.shape, y.copy()))
            self.f = logreg_double.fit(X, y, 'l1', 1.0)

        def predict_log_likelihood_ratio(self, X):
            return logreg_double.predict(self.f, X)

        @property
        def attributes(self):
            return {'parameters': {'coef_': [self.f['coef'].tolist()]}}

    m = arch.get_model(n_obs=100, seed_obs=int(g['seed_obs']))
    bolfire = BOLFIRE(m, 200, seed_marginal=int(g['seed_marginal']), classifier=Host(),
                      bounds={'t1': (-1, 1), 't2': (0, 1)}, n_initial_evidence=2,
                      seed=int(g['seed']))
    bolfire.fit(2, bar=False)
    assert len(seen) == 2
    for t, shape, y in seen:
        assert t is np.ndarray and shape == (400, 17)
        np.testing.assert_array_equal(y, np.r_[np.ones(200), -np.ones(200)])
    ref = g['value_tight'][:2]
    assert np.all(np.abs(bolfire.target_model.Y[:, 0] - ref) <= 1e-7 * (1 + np.abs(ref)))
