"""Conditional device priors (a loc or scale taken from another parameter of the row).

* prior_rvs with per-row loc and scale vectors equals fma(scale, y, loc) of the standard draw y of
  the same stream bit for bit, for every kind; with NULL vectors it equals prior_rvs;
* prior_logpdf with sources matches SciPy with per-row loc / scale (rtol 1e-13, exact infinities
  and NaNs), and the host ModelPrior of M/G/1's hierarchical prior;
* gm_rvs support 4 with every source -1 equals support 3 bit for bit; with M/G/1's sources it
  matches the replay (tests/conditional_prior_replay.py) and keeps t1 <= t2 <= t1 + 10;
* SMC on a small model with a conditional scale is bit-identical when repeated and when sharded.
"""
from functools import partial

import numpy as np
import pytest

import conditional_prior_replay as cr
import prior_replay as pr
from conftest import load_golden

pytestmark = pytest.mark.gpu
SPECS = {'uniform': [0, 0, 1, 0, 0], 'norm': [1, 0, 1, 0, 0], 'truncnorm': [2, -1, 2, 0, 1],
         'expon': [3, 0, 1, 0, 0], 'gamma': [4, 0.7, 0, 1, 0], 'beta': [5, 2, 3, 0, 1]}


def _np(t):
    return t.cpu().numpy()


@pytest.mark.parametrize('kind', sorted(SPECS))
def test_prior_rvs_with_vectors_is_the_affine_step_of_the_standard_draw(kind):
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    B, seed, offset = 3000, 11, 2 ** 32 - 100
    rs = np.random.RandomState(len(kind))
    spec = np.array(SPECS[kind], dtype=np.float64)
    y = _np(ops.prior_rvs(spec, B, seed, offset))                    # loc 0, scale 1: y itself
    loc = rs.uniform(-5, 5, B)
    scale = rs.uniform(0.1, 3, B)
    loc[:6] = [np.nan, 0.0, -0.0, 1e300, -np.inf, 2.0]
    scale[6:14] = [0.0, -0.0, -1.0, np.nan, np.inf, 1e-310, 1e300, 2.0]
    got = _np(ops.prior_rvs(spec, B, seed, offset, loc=dev.to_device(loc), scale=dev.to_device(scale)))
    want = cr.fma(scale, y, loc)
    want[(scale < 0) | np.isnan(scale)] = np.nan
    assert np.array_equal(got, want, equal_nan=True)
    assert got[6] == loc[6] and np.isnan(got[8]) and np.isnan(got[9]) and np.isnan(got[0])
    # only one vector: the other word of the spec
    s2 = spec.copy()
    s2[1 + pr.NSHAPE[kind]], s2[2 + pr.NSHAPE[kind]] = 3.0, 0.5
    got = _np(ops.prior_rvs(s2, B, seed, offset, loc=dev.to_device(loc)))
    assert np.array_equal(got, cr.fma(0.5, y, loc), equal_nan=True)
    got = _np(ops.prior_rvs(s2, B, seed, offset, scale=dev.to_device(np.abs(scale))))
    assert np.array_equal(got, cr.fma(np.abs(scale), y, 3.0), equal_nan=True)
    # the constant path is the same kernel: fma(scale, y, loc) with the spec's words
    assert np.array_equal(_np(ops.prior_rvs(s2, B, seed, offset)), cr.fma(0.5, y, 3.0))


def test_prior_logpdf_with_sources_matches_scipy():
    from elfi_b200 import ops
    rs = np.random.RandomState(4)
    B = 20000
    specs = np.array([[0, 0, 10, 0, 0], [0, 0, 10, 0, 0], [1, 0, 1, 0, 0], [4, 0.7, 0, 1, 0],
                      [5, 2, 3, 0, 4], [2, -1, 2, 0, 1]], dtype=np.float64)
    src = np.array([[-1, -1], [0, -1], [1, 0], [-1, 2], [3, -1], [0, 4]])
    x = np.column_stack([rs.uniform(-1, 11, B), rs.uniform(-1, 21, B), rs.normal(5, 5, B),
                         rs.uniform(-1, 20, B), rs.uniform(-1, 10, B), rs.uniform(-5, 15, B)])
    x[:10, 0] = [0, 10, -0.0, np.nan, np.inf, -1e-300, 1e-300, 5, 5, 5]
    x[10:20, 1] = x[10:20, 0]
    x[20:30, 4] = np.nextafter(x[20:30, 3], -np.inf)
    got = _np(ops.prior_logpdf(x, specs, src))
    want = cr.joint_logpdf(np.concatenate([specs, src], axis=1), x)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    inf = np.isinf(want) | np.isinf(got)
    assert np.array_equal(got[inf], want[inf])
    f = np.isfinite(want)
    assert f.sum() > 500 and inf.sum() > 500
    np.testing.assert_allclose(got[f], want[f], rtol=1e-13, atol=0)
    # every source -1: the bits of the 5-word table
    none = -np.ones_like(src)
    assert np.array_equal(_np(ops.prior_logpdf(x, specs, none)), _np(ops.prior_logpdf(x, specs)),
                          equal_nan=True)


def test_prior_logpdf_matches_host_model_prior_of_mg1():
    from elfi_b200 import ops
    from elfi_b200.examples import mg1
    import elfi_b200 as elfi
    g = load_golden('mg1_prior_logpdf')
    dp = elfi.DeviceModelPrior(mg1.get_model(seed_obs=1), conditional=True)
    got = _np(dp.logpdf(g['x']))
    want = g['logpdf']
    assert np.array_equal(np.isinf(got), np.isinf(want)) and np.array_equal(got[np.isinf(got)],
                                                                          want[np.isinf(want)])
    f = np.isfinite(want)
    np.testing.assert_allclose(got[f], want[f], rtol=1e-13, atol=0)
    assert np.array_equal(_np(ops.prior_logpdf(g['x'], dp.specs, dp.sources)), got)


def _mixture(rs, p, N=200):
    means = rs.uniform(0, 10, (N, p))
    means[:, 1] = means[:, 0] + rs.uniform(-1, 11, N)
    cov = np.diag(rs.uniform(0.5, 4, p))
    w = rs.uniform(0, 1, N)
    return means, cov, w


def test_gm_rvs_support4_without_sources_equals_support3():
    from elfi_b200 import ops
    rs = np.random.RandomState(1)
    for p in (3, 6, 12):
        specs = np.array([[0, -2, 14, 0, 0]] * p, dtype=np.float64)
        specs[2] = [1, 5, 3, 0, 0]
        means, cov, w = _mixture(rs, p)
        a = _np(ops.gm_rvs(means, cov, w, 20000, seed=5, offset=2 ** 32 - 7, support=3, prior=specs))
        b = _np(ops.gm_rvs(means, cov, w, 20000, seed=5, offset=2 ** 32 - 7, support=4, prior=specs,
                           sources=-np.ones((p, 2))))
        assert np.array_equal(a, b), p


def test_gm_rvs_support4_matches_replay_for_mg1():
    from elfi_b200 import ops
    from elfi_b200.examples import mg1
    import elfi_b200 as elfi
    dp = elfi.DeviceModelPrior(mg1.get_model(seed_obs=1), conditional=True)
    rs = np.random.RandomState(2)
    N, B = 300, 20000
    means = np.column_stack([rs.uniform(0, 10, N), np.zeros(N), rs.uniform(0, 0.5, N)])
    means[:, 1] = means[:, 0] + rs.uniform(0, 10, N)
    cov = np.diag([2.0, 4.0, 0.01])
    w = rs.uniform(0, 1, N)
    cdf = ops.gm_cdf(w, N)
    seed, offset = 2 ** 32 + 9, 2 ** 32 - 7
    x = _np(ops.gm_rvs(means, cov, None, B, seed=seed, offset=offset, support=4, prior=dp.specs,
                       sources=dp.sources, cdf=cdf))
    specs7 = np.concatenate([dp.specs, dp.sources], axis=1)
    xr, trial, comp, err, margin = cr.gm_rvs(means, np.linalg.cholesky(cov), _np(cdf), B, seed,
                                             offset, specs7)
    amb = margin < 1e-9
    assert amb.sum() <= max(2, 1e-4 * B), int(amb.sum())
    assert np.all(np.abs(x[~amb] - xr[~amb]) <= err[~amb, None])
    assert np.all(trial >= 0) and np.sum(trial >= 1) > 0.05 * B
    assert np.all((x[:, 1] >= x[:, 0]) & (x[:, 1] <= x[:, 0] + 10))
    assert np.isfinite(cr.joint_logpdf(specs7, x)).all()


def test_smc_with_a_conditional_scale_is_deterministic_and_shard_invariant():
    import elfi_b200 as elfi
    from elfi_b200 import model as em
    from elfi_b200.examples import gauss

    m = em.new_model()
    em.Prior('uniform', 0.5, 3, model=m, name='s')
    em.Prior('norm', 2, m['s'], model=m, name='mu')
    y = np.random.RandomState(3).normal(2.5, 1.5, (1, 20))
    em.Simulator(partial(gauss.gauss_device, n_obs=20), m['mu'], m['s'], observed=y, name='g')
    em.Summary(gauss.ss_mean, m['g'], name='mean')
    em.Summary(gauss.ss_var, m['g'], name='var')
    em.Distance('euclidean', m['mean'], m['var'], name='d')
    dp = elfi.DeviceModelPrior(m, conditional=True)
    np.testing.assert_array_equal(dp.sources, [[-1, 1], [-1, -1]])

    def run(**kw):
        return elfi.SMC(dp.model['d'], batch_size=5000, seed=4, device_proposal=dp, **kw).sample(
            500, quantiles=[0.3, 0.3], bar=False)
    a, b = run(), run()
    assert np.array_equal(a.samples_array, b.samples_array) and np.array_equal(a.weights, b.weights)
    c = run(distributed=False, max_parallel_batches=2)
    d = run(distributed=False, max_parallel_batches=2)
    assert np.array_equal(c.samples_array, d.samples_array) and np.array_equal(c.weights, d.weights)
    assert np.all(np.isfinite(a.weights)) and np.all(a.samples['s'] >= 0.5)
