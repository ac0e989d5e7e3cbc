"""Device AR(1) simulator, its fused distance, and compare_models on device models.

* sim_ar1 element by element against the NumPy replay of its Philox stream (tests/ar1_replay.py),
  within a bound carried through the recursion from the replayed normals' error; row counters
  across 2^32; split launches equal one launch;
* the fused distance and acceptance equal dist_euclid of the materialised series bit for bit;
* the law of x_t given phi, the Rejection posterior against the host model's, the samplers, and
  model choice between AR(1) and MA(2).
"""
import numpy as np
import pytest
import scipy.stats as ss

import ar1_replay as ar

pytestmark = [pytest.mark.gpu, pytest.mark.first_device_run]
PHIS = (-1.0, -0.5, 0.0, 0.9, 1.0)


def _np(t):
    return t.cpu().numpy()


def _phis(B, rs):
    phi = rs.uniform(-1, 1, B)
    phi[:len(PHIS)] = PHIS
    return phi


# ---------------------------------------------------------------------------- sim_ar1
@pytest.mark.parametrize('offset', [0, 2 ** 32 - 300])
@pytest.mark.parametrize('n_obs', [1, 2, 3, 200])
def test_sim_ar1_matches_replay(offset, n_obs):
    from elfi_b200 import ops
    rs = np.random.RandomState(n_obs + offset % 89)
    phi = _phis(1000, rs)
    X, _, _ = ops.sim_ar1(phi, n_obs, seed=7, offset=offset)
    X = _np(X)
    want, err = ar.sim_ar1(phi, n_obs, seed=7, offset=offset)
    bad = ~(np.abs(X - want) <= err)
    assert not bad.any(), (np.argwhere(bad)[:5], np.abs(X - want)[bad][:5], err[bad][:5])
    # a wrong stream would be O(1) off: the bound is tight enough to tell
    assert np.median(err / np.maximum(np.abs(want), 1e-300)) < 1e-11


def test_sim_ar1_split_launches_equal_one_launch():
    from elfi_b200 import ops
    rs = np.random.RandomState(2)
    phi = _phis(1000, rs)
    obs = rs.randn(200) * 2
    base = 2 ** 32 - 400
    whole = ops.sim_ar1(phi, 200, seed=9, offset=base, obs=obs, want_data=True)
    for cut in (1, 400, 777):
        parts = [ops.sim_ar1(phi[:cut], 200, seed=9, offset=base, obs=obs, want_data=True),
                 ops.sim_ar1(phi[cut:], 200, seed=9, offset=base + cut, obs=obs, want_data=True)]
        for j in range(2):
            joined = np.concatenate([_np(parts[0][j]), _np(parts[1][j])])
            assert np.array_equal(joined, _np(whole[j])), (cut, j)


@pytest.mark.parametrize('B', [1, 31, 129, 100003])
def test_fused_distance_equals_dist_euclid_of_the_series(B):
    """Distances and accepted rows of the fused kernel equal dist_euclid of the written series bit
    for bit, at several thresholds, given on the host and on the device, and through the lazy
    output."""
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    from elfi_b200.examples import ar1
    rs = np.random.RandomState(B % 1000)
    phi = _phis(B, rs) if B >= len(PHIS) else rs.uniform(-1, 1, B)
    for n_obs in (1, 2, 200):
        obs = ar1.AR1(0.9, n_obs=n_obs, random_state=np.random.RandomState(1))[0]
        X, d_all, _ = ops.sim_ar1(phi, n_obs, seed=3, offset=2 ** 32 - 1000, obs=obs,
                                  want_data=True)
        want, _ = ops.dist_euclid(X, obs)
        assert np.array_equal(_np(d_all), _np(want)), n_obs
        for q in (0.0, 0.01, 0.5, 1.0):
            thr = float(np.quantile(_np(want), q))
            for t in (thr, dev.to_device(np.array([thr]))):
                _, d, idx = ops.sim_ar1(phi, n_obs, seed=3, offset=2 ** 32 - 1000, obs=obs,
                                        thresholds=t)
                want_d, want_idx = ops.dist_euclid(X, obs, thresholds=t)
                assert np.array_equal(_np(d), _np(want_d)), (n_obs, q)
                assert np.array_equal(_np(idx), _np(want_idx)), (n_obs, q)
    lazy = ar1.ar1_device(phi, n_obs=200, batch_size=B, random_state=np.random.RandomState(4))
    obs = rs.randn(200)
    d, idx = lazy.euclidean(dev.to_device(obs), 15.0)
    want_d, want_idx = ops.dist_euclid(lazy.materialize(), obs, thresholds=15.0)
    assert np.array_equal(_np(d), _np(want_d)) and np.array_equal(_np(idx), _np(want_idx))


# ---------------------------------------------------------------------------- statistics
@pytest.mark.parametrize('phi', PHIS)
def test_law_given_phi(phi):
    """x_t / s_t ~ N(0, 1) with s_t^2 = sum_{k<t} phi^(2k), the exact law of x_t given phi."""
    from elfi_b200 import ops
    B = 20000
    X = _np(ops.sim_ar1(np.full(B, phi), 200, seed=11)[0])
    for t in (1, 2, 10, 200):
        s = np.sqrt(np.sum(phi ** (2 * np.arange(t))))
        p = ss.kstest(X[:, t - 1] / s, 'norm').pvalue
        assert p > 1e-4, (phi, t, p)


def test_device_rejection_posterior_matches_host():
    """Tolerance: the posterior means of the two modes differ by less than 4 standard errors of
    their difference.  The modes draw from the same law through different generators, so their
    samples are independent; the host sample is the smaller one and dominates the error."""
    import elfi_b200 as elfi
    from elfi_b200.examples import ar1
    host_m = ar1.get_model(seed_obs=2)
    res_h = elfi.Rejection(host_m['d'], batch_size=10000, seed=1).sample(300, quantile=0.01,
                                                                          bar=False)
    m, dp = ar1.get_device_model(seed_obs=2)
    assert np.array_equal(m.observed['AR1'], host_m.observed['AR1'])
    res_d = elfi.Rejection(m['d'], batch_size=100000, seed=1).sample(3000, quantile=0.01,
                                                                      bar=False)
    h, d = res_h.samples['phi'], res_d.samples['phi']
    se = np.sqrt(h.var() / len(h) + d.var() / len(d))
    assert abs(h.mean() - d.mean()) < 4 * se, (h.mean(), d.mean(), se)


# ---------------------------------------------------------------------------- samplers
def test_device_model_smc_and_adaptive_distance_smc():
    import elfi_b200 as elfi
    from elfi_b200.examples import ar1
    m, dp = ar1.get_device_model(seed_obs=3)

    def run(**kw):
        return elfi.SMC(m['d'], batch_size=10000, seed=4, device_proposal=dp, **kw).sample(
            1000, quantiles=[0.1, 0.3, 0.3], bar=False)
    smc = run()
    assert len(smc.populations) == 3 and np.all(np.isfinite(smc.weights))
    assert np.all(np.abs(smc.samples['phi']) <= 1)
    m['d'].become(elfi.AdaptiveDistance(m['AR1']))
    ad = elfi.AdaptiveDistanceSMC(m['d'], batch_size=10000, seed=5, device_proposal=dp).sample(
        1000, rounds=3, quantile=0.3, bar=False)
    assert len(ad.populations) == 3
    assert np.all(np.isfinite(ad.samples_array))


# ---------------------------------------------------------------------------- model choice
def _autocov(x, lag):
    """Autocovariance at `lag` of the series: lazy simulator output is materialised."""
    from elfi_b200 import ops
    from elfi_b200.throughput import LazySimulation
    if isinstance(x, LazySimulation):
        x = x.materialize()
    return ops.autocov(np.atleast_2d(x) if not hasattr(x, 'is_cuda') else x, lags=(lag,))[:, 0]


def test_compare_models_prefers_ar1_over_ma2_on_an_ar1_series():
    import elfi_b200 as elfi
    from elfi_b200.examples import ar1, ma2
    n_obs = 100
    y = ar1.AR1(0.9, n_obs=n_obs, random_state=np.random.RandomState(5))

    def task(sim, priors):
        m = elfi.new_model()
        for name, lo, width in priors:
            elfi.Prior('uniform', lo, width, model=m, name=name)
        elfi.Simulator(sim, *[m[p[0]] for p in priors], observed=y, name='Y')
        elfi.Summary(_autocov, m['Y'], 1, name='S1')
        elfi.Summary(_autocov, m['Y'], 2, name='S2')
        elfi.Distance('euclidean', m['S1'], m['S2'], name='d')
        return m
    m_ar = task(lambda phi, batch_size=1, random_state=None: ar1.ar1_device(
        phi, n_obs=n_obs, batch_size=batch_size, random_state=random_state), [('phi', -1, 2)])
    m_ma = task(lambda t1, t2, batch_size=1, random_state=None: ma2.MA2_device(
        t1, t2, n_obs=n_obs, batch_size=batch_size, random_state=random_state),
        [('t1', -2, 4), ('t2', -1, 2)])
    res = [elfi.Rejection(m['d'], batch_size=100000, seed=6).sample(1000, quantile=0.01,
                                                                       bar=False)
           for m in (m_ar, m_ma)]
    p = elfi.compare_models(res)
    assert p.shape == (2,) and abs(p.sum() - 1) < 1e-12
    assert p[0] > p[1], p


def test_compare_models_reference_three_model_test_on_host_models():
    """The reference's test_compare_models: gauss, gauss with a wider prior on mu, and an MA2
    simulator in its place."""
    import elfi_b200 as elfi
    from elfi_b200.examples import gauss, ma2
    m = gauss.get_model(seed_obs=6)
    res1 = elfi.Rejection(m['d'], seed=7).sample(100, bar=False)
    m['mu'].become(elfi.Prior('uniform', -10, 50))
    res2 = elfi.Rejection(m['d'], seed=8).sample(100, bar=False)
    m['gauss'].become(elfi.Simulator(ma2.MA2, m['mu'], m['sigma'], observed=m.observed['gauss']))
    res3 = elfi.Rejection(m['d'], seed=9).sample(100, bar=False)
    p = elfi.compare_models([res1, res2, res3])
    assert p[0] > p[1]
    assert p[1] > p[2]
