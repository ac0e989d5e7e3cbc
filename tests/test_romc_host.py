"""ROMC's host-model path under the CPU double of the C ABI reproduces the unmodified reference
(tests/golden/gen_golden_romc.py): nuisances, starting points, Nelder-Mead results, Hessians,
rotations and box limits bit for bit; surrogate coefficients and weights to 1e-10 (1 + |v|)."""
import numpy as np
import pytest

import elfi_b200
import romc_cases
import abi_double
import romc_double
from elfi_b200 import device as dev, ops, romc
from elfi_b200.examples import ma2


def _close(a, b, tol=1e-10):
    a, b = np.asarray(a, dtype=float), np.asarray(b, dtype=float)
    assert a.shape == b.shape
    assert np.all(np.abs(a - b) <= tol * (1 + np.abs(b)))


def _case(name):
    if name == 'oned':
        m, dname = romc_cases.one_d_model(elfi_b200)
        return romc.ROMC(m[dname], [(-2.5, 2.5)]), 100, 21
    m = ma2.get_model(n_obs=50, true_params=[.6, .2], seed_obs=3)
    return romc.ROMC(m['d'], [(-2, 2), (-1, 1)]), 20, 5


@pytest.mark.parametrize('name', ['oned', 'ma2'])
def test_host_path_matches_reference(cpu_double, monkeypatch, golden, name):
    abi_double.install(monkeypatch, romc_double.TABLE)
    g = {k[len(name) + 1:]: v for k, v in golden('romc').items() if k.startswith(name + '_')}
    r, n1, seed = _case(name)
    assert not r.on_device
    r.solve_problems(n1=n1, seed=seed)
    np.testing.assert_array_equal(r.nuisance, g['nuisance'])
    np.testing.assert_array_equal(r.x0, g['x0'])
    np.testing.assert_array_equal(r.x_min, g['x_min'])
    np.testing.assert_array_equal(r.f_min, g['f_min'])
    np.testing.assert_array_equal(r.solved, g['success'])
    np.testing.assert_array_equal(r.nit, g['nit'])
    np.testing.assert_array_equal(r.nfev, g['nfev'])
    np.testing.assert_array_equal(r.hess[r.solved], g['hess'])
    r.estimate_regions(eps_filter=float(g['eps']), fit_models=True)
    np.testing.assert_array_equal(r.accepted, g['accepted'])
    np.testing.assert_array_equal(r.rotation, g['rotation'])
    np.testing.assert_array_equal(r.center, g['center'])
    np.testing.assert_array_equal(r.limits, g['limits'])
    # the objectives at the reference's fitting points, and the fits on them
    y = dev.to_host(r._evaluate_regions(g["fit_x"]))
    np.testing.assert_array_equal(y, g['fit_y'])
    coef = np.array([romc.fit_local_model(x, yy) for x, yy in zip(g['fit_x'], g['fit_y'])])
    _close(coef, g['coef'])
    # distances (the local surrogates) and weights at the reference's draws
    S = g['samples']
    R, n2, p = S.shape
    dist = np.array([[romc_double.quad(S[k, j], g['coef'][k]) for j in range(n2)]
                     for k in range(R)])
    _close(dist.reshape(-1), g['distances'])
    q = np.array([[1.0 / r.volume[k] if romc_double.contains(S[k, j], r.rotation_inv[k],
                                                            r.center[k], r.limits[k]) else 0.0
                   for j in range(n2)] for k in range(R)])
    pr = dev.to_host(r._prior_pdf(S.reshape(-1, p))).reshape(R, n2)
    w = dev.to_host(ops.romc_weights(g["distances"].reshape(R, n2), pr, q, r.eps_cutoff))
    _close(w, g['weights'])


def test_reference_functional_example(cpu_double, monkeypatch):
    """The reference's test_romc1 assertions on its one-parameter example."""
    abi_double.install(monkeypatch, romc_double.TABLE)
    m, dname = romc_cases.one_d_model(elfi_b200)
    r = romc.ROMC(m[dname], [(-2.5, 2.5)])
    r.solve_problems(n1=100, seed=21)
    r.estimate_regions(eps_filter=.75, fit_models=True, fit_models_args={'nof_points': 30})
    r.sample(n2=30, seed=3)
    assert np.allclose(r.compute_expectation(h=lambda x: np.squeeze(x)), 0, atol=.4)
    assert np.allclose(r.compute_expectation(h=lambda x: np.squeeze(x) ** 2), 1.1, atol=.4)
    assert r.compute_ess() > 100
    res = r.extract_result()
    assert res.outputs['theta'].shape == (r.samples.shape[0] * 30,)
    x = np.linspace(-2.5, 2.5, 7)[:, None]
    un = r.eval_unnorm_posterior(x)
    want = romc_double.posterior_unnorm(x, r.prior.pdf(x).reshape(-1), r.eps_cutoff, r.center,
                                        r.rotation_inv, r.limits, r.coef)
    np.testing.assert_array_equal(un, want)
    assert np.isfinite(r.compute_divergence(lambda t: np.exp(-0.5 * t[:, 0] ** 2), step=0.5))


def test_argument_errors(cpu_double, monkeypatch):
    abi_double.install(monkeypatch, romc_double.TABLE)
    m, dname = romc_cases.one_d_model(elfi_b200)
    with pytest.raises(NotImplementedError):
        romc.ROMC(m[dname], custom_optim_class=object)
    with pytest.raises(ValueError):
        romc.ROMC(m)
    r = romc.ROMC(m[dname], [(-2.5, 2.5)])
    with pytest.raises(ValueError):
        r.compute_eps(0.5)
    with pytest.raises(NotImplementedError):
        r.solve_problems(5, use_bo=True)
    with pytest.raises(NotImplementedError):
        r.solve_problems(5, optimizer_args={'method': 'BFGS'})
    with pytest.raises(ValueError):
        r.solve_problems(0)
    with pytest.raises(ValueError):
        r.sample(3)
    r.solve_problems(4, seed=1)
    with pytest.raises(NotImplementedError):
        r.estimate_regions(1.0, use_surrogate=True)
    with pytest.raises(ValueError):
        r.compute_eps(1.5)
    with pytest.raises(NotImplementedError):
        r.visualize_region(0)
    with pytest.raises(ValueError):
        ops.RomcNelderMead(np.zeros((3, 17)))


@pytest.mark.parametrize('case', ['p1_narrow', 'p2_narrow', 'p3_mixed', 'p5_wide', 'p5_narrow'])
def test_local_fit_matches_reference_linear_regression(golden, case):
    """The reference's surrogate fit on boxes where singular values fall below scikit-learn's cutoff
    (narrow sides) or the problem is underdetermined (p = 5: 21 coefficients, 20 points)."""
    g = golden('romc_fits')
    _close(romc.fit_local_model(g[case + '_x'], g[case + '_y']), g[case + '_coef'])


def test_unnorm_posterior_without_local_models(cpu_double, monkeypatch):
    """Without local models a region counts where its own objective is <= eps (no containment),
    as RomcPosterior._sum_over_indicators; only the regions' columns of each batch are kept."""
    abi_double.install(monkeypatch, romc_double.TABLE)
    m, dname = romc_cases.one_d_model(elfi_b200)
    r = romc.ROMC(m[dname], [(-2.5, 2.5)])
    r.solve_problems(n1=20, seed=4)
    r.estimate_regions(eps_filter=.75, fit_models=False)
    x = np.array([[-1.2], [0.1], [0.9]])
    f = np.array([[dev.to_host(r._evaluate(np.full((20, 1), t[0])))[i] for i in r.region_problem]
                  for t in x])
    want = r.prior.pdf(x).reshape(-1) * np.sum(f <= r.eps_cutoff, axis=1)
    np.testing.assert_array_equal(r.eval_unnorm_posterior(x), want)
