"""ROMC kernels on the device against scipy and the NumPy restatement (tests/romc_double.py), and
ROMC end to end on the device MA2 model."""
import numpy as np
import pytest
import scipy.optimize as so
import scipy.stats as ss

import romc_double
from elfi_b200 import device as dev, ops, romc
from elfi_b200.examples import ma2

pytestmark = pytest.mark.gpu


def _objective(kind, x):
    x = np.atleast_2d(x)
    if kind == 'rosen':
        return np.sum(100.0 * (x[:, 1:] - x[:, :-1] ** 2) ** 2 + (1 - x[:, :-1]) ** 2, axis=1)
    if kind == 'steps':           # piecewise constant: ties in fsim
        return np.sum(np.floor(4 * np.abs(x - 0.3)), axis=1)
    if kind == 'nan':
        f = np.sum((x - 0.5) ** 2, axis=1)
        return np.where(x[:, 0] > 1.2, np.nan, f)
    return np.sum((np.arange(1, x.shape[1] + 1) * (x - 0.25)) ** 2, axis=1)


def _scipy(kind, x0, monkeypatch, stable):
    if stable:     # the kernels' stable vertex order (NumPy's SIMD sort is not stable for p >= 3)
        monkeypatch.setattr(np, 'argsort', lambda a, *k, **kw: np.lexsort(
            (np.arange(len(a)), np.where(np.isnan(a), 0.0, a), np.isnan(a))))
    try:
        return [so.minimize(lambda x: float(_objective(kind, x)[0]), x, method='Nelder-Mead')
                for x in x0]
    finally:
        monkeypatch.undo()


@pytest.mark.parametrize('p,n,kind', [(1, 1000, 'quad'), (2, 1000, 'rosen'), (2, 1000, 'steps'),
                                      (2, 300, 'nan'), (5, 1000, 'quad'), (16, 1000, 'quad')])
def test_nm_step_equals_scipy(monkeypatch, p, n, kind):
    x0 = np.random.RandomState(p).uniform(-1.5, 1.5, (n, p))
    nm = ops.RomcNelderMead(x0)
    while nm.running():
        nm.step(_objective(kind, dev.to_host(nm.theta)))
    x_min, f_min, nit, nfev, success = nm.result()
    for i, r in enumerate(_scipy(kind, x0, monkeypatch, stable=p > 2)):
        np.testing.assert_array_equal(x_min[i], r.x)
        np.testing.assert_array_equal(f_min[i], r.fun)
        assert (nit[i], nfev[i], success[i]) == (r.nit, r.nfev, r.success)


def _host_romc(name, g):
    """A host-model ROMC whose objectives are the golden case's (its nuisances)."""
    import elfi_b200
    import romc_cases
    if name == 'oned':
        m, dname = romc_cases.one_d_model(elfi_b200)
        r = romc.ROMC(m[dname], [(-2.5, 2.5)])
    else:
        m = ma2.get_model(n_obs=50, true_params=[.6, .2], seed_obs=3)
        r = romc.ROMC(m['d'], [(-2, 2), (-1, 1)])
    r.n1, r.nuisance = len(g['x_min']), g['nuisance']
    return r


@pytest.mark.parametrize('name', ['oned', 'ma2'])
def test_line_search_equals_golden(golden, name):
    """The device line search along the reference's rotations (columns of a real rotation and both
    sides at p = 2) reproduces its box limits bit for bit."""
    g = {k[len(name) + 1:]: v for k, v in golden('romc').items() if k.startswith(name + '_')}
    acc = g['accepted']
    x_min = g['x_min']
    p = x_min.shape[1]
    rot = np.broadcast_to(np.eye(p), (len(x_min), p, p)).copy()
    rot[acc] = g['rotation']
    ls = ops.RomcLineSearch(x_min, rot, acc, float(g['eps']))
    r = _host_romc(name, g)
    while ls.running():
        rows = dev.to_host(ls.istate[:, 2]).reshape(2 * p, -1) == 0
        ls.step(np.stack([dev.to_host(r._evaluate(ls.theta[k], rows[k])) for k in range(2 * p)]))
    np.testing.assert_array_equal(romc.secure_limits(ls.limits()[acc]), g['limits'])


def _boxes(R, p, seed):
    rs = np.random.RandomState(seed)
    center = rs.randn(R, p)
    rot = np.array([np.linalg.qr(rs.randn(p, p))[0] for _ in range(R)])
    lim = np.stack([-rs.uniform(0.1, 1, (R, p)), rs.uniform(0.1, 1, (R, p))], -1)
    vol = np.prod(lim[:, :, 1] - lim[:, :, 0], axis=1)
    coef = rs.randn(R, 1 + p + p * (p + 1) // 2)
    return center, rot, np.linalg.inv(rot), lim, vol, coef


@pytest.mark.parametrize('p', [1, 2, 5, 16])
def test_box_sample_and_weights(p):
    center, rot, rinv, lim, vol, coef = _boxes(6, p, p)
    pts, q, surr = ops.romc_box_sample(center, rot, rinv, lim, vol, 4000, seed=11, coef=coef)
    pts, q, surr = dev.to_host(pts), dev.to_host(q), dev.to_host(surr)
    for r in range(6):
        u = np.einsum('ij,nj->ni', rinv[r], pts[r] - center[r])
        lo, hi = lim[r, :, 0], lim[r, :, 1]
        assert np.all(u >= lo - 1e-9 * (1 + abs(lo))) and np.all(u <= hi + 1e-9 * (1 + abs(hi)))
        for d in range(p):
            assert ss.kstest((u[:, d] - lo[d]) / (hi[d] - lo[d]), 'uniform').pvalue > 1e-4
    ref_p, ref_q, ref_s = romc_double.box_sample(center, rot, rinv, lim, vol, 50, 11, coef)
    np.testing.assert_allclose(pts[:, :50], ref_p, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(surr[:, :50], ref_s, rtol=1e-12, atol=1e-12)
    dist = np.abs(surr)
    prior = np.random.RandomState(1).uniform(0, 2, q.shape)
    w = dev.to_host(ops.romc_weights(dist, prior, q, 1.0))
    np.testing.assert_allclose(w, romc_double.weights(dist, prior, q, 1.0), rtol=1e-12, atol=0)


@pytest.mark.parametrize('p', [1, 2, 5])
def test_posterior_unnorm(p):
    R = 40
    center, rot, rinv, lim, vol, coef = _boxes(R, p, 100 + p)
    theta = np.random.RandomState(p).randn(3000, p)
    prior = np.random.RandomState(2).uniform(0, 1, len(theta))
    got = dev.to_host(ops.romc_posterior_unnorm(theta, prior, 0.5, center, rinv, lim, coef))
    want = romc_double.posterior_unnorm(theta, prior, 0.5, center, rinv, lim, coef)
    # points within 1e-12 of a box face may fall either way (NumPy's dot sums in another order)
    near = np.zeros(len(theta), dtype=bool)
    for k in range(R):
        u = np.einsum('ij,nj->ni', rinv[k], theta - center[k])
        gap = np.minimum(np.abs(u - lim[k, :, 0]), np.abs(u - lim[k, :, 1]))
        near |= np.any(gap <= 1e-12 * (1 + np.abs(u)), axis=1)
    np.testing.assert_array_equal(got[~near], want[~near])
    fv = np.random.RandomState(3).uniform(0, 1, (len(theta), R))
    got = dev.to_host(ops.romc_posterior_unnorm(theta, prior, 0.5, fvals=fv))
    np.testing.assert_array_equal(got, prior * np.sum(fv <= 0.5, axis=1))


def _device_ma2():
    return ma2.get_device_model(n_obs=100, true_params=[.6, .2], seed_obs=4)


def _check_rows(r, th):
    """Row i's objective is the same bits when the other rows change and when n1 changes."""
    n = len(th)
    r.n1, r._sim_seed = n, 17
    a = dev.to_host(r._evaluate(th))
    th2 = th.copy()
    th2[1::2] = th[::-1][1::2]
    b = dev.to_host(r._evaluate(th2))
    np.testing.assert_array_equal(a[::2], b[::2])
    r.n1 = n // 3
    np.testing.assert_array_equal(dev.to_host(r._evaluate(th[:n // 3])), a[:n // 3])
    assert np.all(np.isfinite(a)) and len(np.unique(a)) > n // 2


def test_row_invariance_ma2():
    m = _device_ma2()
    r = romc.ROMC(m['d'], [(-2, 2), (-1, 1)], device_prior=ma2.DeviceProposal)
    assert r.on_device
    rs = np.random.RandomState(0)
    _check_rows(r, np.column_stack([rs.uniform(-1, 1, 600), rs.uniform(-.5, .5, 600)]))


def test_row_invariance_gnk():
    from elfi_b200.examples import gnk
    m, proposal = gnk.get_device_model(n_obs=100, seed=2, summary='ss_robust')
    r = romc.ROMC(m['d'], [(0, 10)] * 4, device_prior=proposal)
    assert r.on_device
    _check_rows(r, np.random.RandomState(1).uniform(0.5, 5, (600, 4)))


def romc_vs_rejection(seed):
    """ROMC posterior mean - rejection posterior mean per parameter on the device MA2 model:
    ROMC with n1 = 10000, eps the 0.1 quantile, local models, n2 = 50; rejection keeps the best
    5000 of 5e6 simulations.  Both seeded from `seed`."""
    import elfi_b200
    r = romc.ROMC(_device_ma2()['d'], [(-2, 2), (-1, 1)], device_prior=ma2.DeviceProposal)
    r.solve_problems(n1=10000, seed=3 + 10 * seed)
    r.estimate_regions(eps_filter=float(r.compute_eps(0.1)), fit_models=True)
    r.sample(n2=50, seed=4 + 10 * seed)
    mean = np.array([r.compute_expectation(lambda x: x[..., k]) for k in range(2)])
    rej = elfi_b200.Rejection(_device_ma2()['d'], batch_size=100000, seed=5 + 10 * seed)
    res = rej.sample(5000, quantile=0.001)
    ref = np.array([np.mean(res.samples['t1']), np.mean(res.samples['t2'])])
    return mean - ref


# ROMC mean - rejection mean (t1, t2) for seeds 0 .. 4, measured on an NVIDIA H100 80GB HBM3 with
# romc_vs_rejection: ROMC's t2 mean lies below rejection's by 0.02 to 0.10 on every seed
E2E_SPREAD = np.array([[-0.0000191, -0.0672928], [0.0324540, -0.0209305], [0.0209707, -0.0957591],
                       [0.0260526, -0.0966819], [0.0349278, -0.0387805]])
E2E_TOL = 1.5 * np.max(np.abs(E2E_SPREAD), axis=0)        # 0.052 for t1, 0.145 for t2


def test_device_ma2_end_to_end():
    """The ROMC posterior mean on the device MA2 model against a long rejection run on the same
    data, within 1.5 times the largest deviation seen over five seeds (E2E_SPREAD)."""
    diff = romc_vs_rejection(0)
    print('ROMC - rejection', diff)
    assert np.all(np.abs(diff) < E2E_TOL)
