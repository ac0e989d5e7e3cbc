"""Bodies of the Distance('mahalanobis', VI=...) sampler tests (shared by the CPU-double and GPU
collections): the host MA2 model with a Mahalanobis distance node against the reference's runs
(tests/golden/gen_golden_mahalanobis.py)."""
import numpy as np

from conftest import load_golden

RUNS = ('quantile', 'nsim', 'threshold')
REJECTION = {'quantile': (dict(batch_size=1000, seed=123), dict(n_samples=100, quantile=0.01)),
             'nsim': (dict(batch_size=500, seed=7), dict(n_samples=64, n_sim=3000)),
             'threshold': (dict(batch_size=1000, seed=123), dict(n_samples=150, threshold=0.3))}
SMC = (dict(batch_size=1000, seed=20), dict(n_samples=150, thresholds=[1.0, 0.5]))
RTOL, ATOL = 1e-6, 1e-9   # the SMC parity bar of tests/test_samplers_gpu.py
D_MAX = 192               # include/elfi_b200.h, ELFI_B200_MAHALANOBIS_D_MAX
DIMS = (1, 2, 3, 5, 16, 31, 32, 33, 64, 100, 145, 160, D_MAX)
KINDS = ('symmetric', 'nonsymmetric', 'indefinite')


def make_vi(kind, D, rs):
    """A (D, D) VI: SPD; SPD plus an antisymmetric part (u'VIu > 0, VI != VI'); or symmetric with
    eigenvalues of alternating sign, the first negative, so that rows with q < 0 (NaN) occur."""
    A = rs.randn(D, D)
    spd = A @ A.T / D + np.eye(D)
    if kind == 'symmetric':
        return spd
    if kind == 'nonsymmetric':
        return spd + 0.5 * (A - A.T) / np.sqrt(D)
    Q = np.linalg.qr(A)[0]
    return (Q * np.where(np.arange(D) % 2, 1.0, -1.0)) @ Q.T


def make_rows(B, D, rs, obs):
    """B rows of summaries around obs with a NaN, a +inf, a -inf, an exact copy of obs and a row of
    -0.0 among the first ones (as far as B allows)."""
    S = obs + rs.randn(B, D) * rs.uniform(0.1, 5)
    special = [(0, np.nan), (1, np.inf), (2, -np.inf)]
    for i, v in special[:B]:
        S[i, (7 * i) % D] = v
    if B > 3:
        S[3] = obs
    if B > 4:
        S[4] = -0.0
    return S


def same_bits(a, b):
    """Equal bit patterns, NaN positions included."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and bool(np.all((a.view(np.uint64) == b.view(np.uint64)) |
                                              (np.isnan(a) & np.isnan(b))))


def case_node_in_a_model():
    """Distance('mahalanobis', S1, S2, VI=...) inside the MA2 model == cdist over the stacked
    summaries bit for bit."""
    from scipy.spatial.distance import cdist

    import elfi_b200 as elfi
    from elfi_b200 import device as dev
    from elfi_b200.examples import ma2
    m = ma2.get_model(seed_obs=4)
    VI = np.array([[2.0, 0.3], [-0.1, 0.5]])
    elfi.Distance('mahalanobis', m['S1'], m['S2'], VI=VI, name='dm')
    out = m.generate(700, ['S1', 'S2', 'dm'], seed=5)
    S = np.column_stack([dev.to_host(out['S1']), dev.to_host(out['S2'])])
    obs = np.array([float(dev.to_host(m[k].observed).ravel()[0]) for k in ('S1', 'S2')])
    assert same_bits(dev.to_host(out['dm']), cdist(S, obs[None], 'mahalanobis', VI=VI).ravel())


def model(g):
    import elfi_b200 as elfi
    from elfi_b200.examples import ma2
    m = ma2.get_model(seed_obs=4)
    m['d'].become(elfi.Distance('mahalanobis', m['S1'], m['S2'], VI=g['VI']))
    return m


def case_pilot():
    """The fixture's VI is the inverse covariance of the seeded pilot, which this model draws too."""
    from elfi_b200 import device as dev
    from elfi_b200.examples import ma2
    g = load_golden('ma2_mahalanobis')
    out = ma2.get_model(seed_obs=4).generate(int(g['pilot_n']), ['S1', 'S2'],
                                             seed=int(g['pilot_seed']))
    pilot = np.column_stack([dev.to_host(out[k]).ravel() for k in ('S1', 'S2')])
    assert np.array_equal(pilot, g['pilot'])
    assert np.array_equal(np.linalg.inv(np.cov(pilot, rowvar=False)), g['VI'])


def case_rejection(run):
    """Rejection in quantile, n_sim and threshold mode: bit for bit."""
    import elfi_b200 as elfi
    g = load_golden('ma2_mahalanobis')
    init, kw = REJECTION[run]
    res = elfi.Rejection(model(g)['d'], **init).sample(bar=False, **kw)
    pre = run + '_'
    assert res.n_sim == int(g[pre + 'n_sim'])
    assert res.threshold == float(g[pre + 'threshold'])
    assert np.array_equal(res.discrepancies, g[pre + 'd'])
    for k in ('t1', 't2'):
        assert np.array_equal(res.samples[k], g[pre + k]), k


def case_smc():
    """SMC with two thresholds: the first population bit for bit, then the SMC parity bar."""
    import elfi_b200 as elfi
    g = load_golden('ma2_mahalanobis')
    res = elfi.SMC(model(g)['d'], **SMC[0]).sample(bar=False, **SMC[1])
    assert res.n_sim == int(g['smc_n_sim'])
    assert len(res.populations) == int(g['smc_n_pops'])
    for i, pop in enumerate(res.populations):
        pre = 'pop{}_'.format(i)
        assert pop.n_sim == int(g[pre + 'n_sim']), i
        got = {'t1': pop.samples['t1'], 't2': pop.samples['t2'], 'd': pop.discrepancies}
        for k, v in got.items():
            if i == 0:
                assert np.array_equal(v, g[pre + k]), (i, k)
            else:
                np.testing.assert_allclose(v, g[pre + k], rtol=RTOL, atol=ATOL, err_msg=(i, k))
        np.testing.assert_allclose(pop.weights, g[pre + 'weights'], rtol=1e-5)
        np.testing.assert_allclose(pop.threshold, float(g[pre + 'threshold']), rtol=1e-7)
    np.testing.assert_allclose(res.samples['t1'], g['smc_t1'], rtol=RTOL, atol=ATOL)
    np.testing.assert_allclose(res.discrepancies, g['smc_d'], rtol=RTOL, atol=ATOL)
    np.testing.assert_allclose(res.weights, g['smc_weights'], rtol=1e-5)
    np.testing.assert_allclose(res.threshold, float(g['smc_threshold']), rtol=1e-7)
