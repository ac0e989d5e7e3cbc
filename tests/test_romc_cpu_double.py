"""The NumPy restatement of the lock-step Nelder-Mead (tests/romc_double.py) equals
scipy.optimize.minimize(method='Nelder-Mead') problem by problem, and NumPy's argsort order of
tied and NaN objective values is the kernels' stable order for p <= 2."""
import itertools

import numpy as np
import pytest
import scipy.optimize as so

import romc_double
from test_romc_gpu import _objective, _scipy


def _run(kind, x0, maxiter=None):
    st, ist, th = romc_double.nm_init(x0)
    p = x0.shape[1]
    mi = 200 * p if maxiter is None else maxiter
    while (ist[:, 0] != romc_double.DONE).any():
        romc_double.nm_step(st, ist, _objective(kind, th), th, mi, 200 * p)
    return st[:, :p], st[:, -1], ist[:, 1], ist[:, 2], ist[:, 4] == 0


@pytest.mark.parametrize('p,kind', [(1, 'quad'), (2, 'rosen'), (2, 'steps'), (2, 'nan'),
                                    (5, 'quad'), (5, 'rosen'), (5, 'steps'), (16, 'quad')])
def test_restatement_equals_scipy(monkeypatch, p, kind):
    x0 = np.random.RandomState(10 + p).uniform(-1.5, 1.5, (12 if p < 16 else 3, p))
    x_min, f_min, nit, nfev, ok = _run(kind, x0)
    for i, r in enumerate(_scipy(kind, x0, monkeypatch, stable=p > 2)):
        np.testing.assert_array_equal(x_min[i], r.x)
        np.testing.assert_array_equal(f_min[i], r.fun)
        assert (nit[i], nfev[i], ok[i]) == (r.nit, r.nfev, r.success)


def test_maxiter_stop():
    x0 = np.random.RandomState(0).uniform(-1.5, 1.5, (4, 2))
    _, _, nit, _, ok = _run('rosen', x0, maxiter=7)
    assert np.all(nit == 7) and not ok.any()
    for i, x in enumerate(x0):
        r = so.minimize(lambda y: float(_objective('rosen', y)[0]), x, method='Nelder-Mead',
                        options={'maxiter': 7})
        assert r.nit == 7 and not r.success


@pytest.mark.parametrize('n', [2, 3])
def test_numpy_argsort_is_stable_for_p_le_2(n):
    for a in itertools.product([0., 1., np.inf, np.nan], repeat=n):
        a = np.array(a)
        np.testing.assert_array_equal(np.argsort(a), romc_double._stable_order(a))
