"""CPU checks of the n-D Gaussian mean model (gauss.get_model(nd_mean=True)).

* the NumPy statement of the three entry points (tests/gauss_nd_double.py) against np.mean, np.var
  and np.sum directly, including the switch of order between D = 1 and D >= 2 and the distance's
  switch at D = 8;
* the NumPy replay of the simulator's Philox stream (tests/gauss_nd_replay.py);
* on the CPU test double extended by the statement: the unmodified host code reproduces the
  reference's goldens (tests/golden/gen_golden_gauss_nd.py) bit for bit, SMC at the SMC parity bar;
  argument errors; the lazy output of the device model and its dispatch.
"""
import numpy as np
import pytest

from conftest import load_golden
from mahalanobis_cases import ATOL, RTOL, same_bits

DIMS = (1, 2, 3, 7, 8, 9, 16, 33)
NOBS = (1, 2, 15, 50, 1000)
DIST_DIMS = (1, 7, 8, 9, 16, 127, 128, 129, 300)
CONFIGS = {'d1': ([4], [1]), 'd2': ([4, 4], [[1, .5], [.5, 1]]), 'd5': ([1, 2, 3, 4, 5], None)}
SEED_OBS = {'d1': 3, 'd2': 4, 'd5': 5}
THRESHOLD = {'d1': 0.5, 'd2': 1.0, 'd5': 3.5}
SMC_THRESHOLDS = {'d1': [1.0, 0.5], 'd2': [2.0, 1.0], 'd5': [4.0, 3.0]}
REJECTION = {'quantile': (dict(batch_size=1000, seed=123), dict(n_samples=100, quantile=0.01)),
             'nsim': (dict(batch_size=500, seed=7), dict(n_samples=64, n_sim=3000)),
             'threshold': (dict(batch_size=1000, seed=123), dict(n_samples=150))}


def crafted(B, n, D, rs):
    """(B, n, D) data of wide dynamic range, with NaN, +inf, -inf and a row of -0.0."""
    y = rs.randn(B, n, D) * np.exp(rs.randn(B, n, D) * 4)
    y[0, n // 2, 0] = np.nan
    y[1, 0, D - 1] = np.inf
    y[2, n - 1, 0] = -np.inf
    y[3] = -0.0
    return y


# ---------------------------------------------------------------------------- the NumPy statement
@pytest.mark.parametrize('D', DIMS)
def test_statement_equals_numpy(D):
    import gauss_nd_double as g
    rs = np.random.RandomState(D)
    for n in NOBS:
        y = crafted(6, n, D, rs)
        mean, var = g.meanvar(y)
        with np.errstate(invalid='ignore'):
            assert same_bits(mean, np.mean(y, axis=1)), n
            assert same_bits(var, np.var(y, axis=1)), n
            assert same_bits(g.axis1_sum(y), np.sum(y, axis=1)), n


def test_statement_order_switches_at_d_two():
    """D = 1 sums pairwise, D >= 2 folds: each order is needed (the other one differs)."""
    import gauss_nd_double as g
    rs = np.random.RandomState(1)
    y = rs.randn(200, 1000, 1) * np.exp(rs.randn(200, 1000, 1) * 4)
    fold = np.zeros(200)
    for t in range(1000):
        fold = fold + y[:, t, 0]
    assert same_bits(g.axis1_sum(y)[:, 0], np.sum(y, axis=1)[:, 0])
    assert not np.array_equal(fold, np.sum(y, axis=1)[:, 0])
    y2 = np.repeat(y, 2, axis=2)
    assert same_bits(g.axis1_sum(y2), np.sum(y2, axis=1))
    assert np.array_equal(g.axis1_sum(y2)[:, 0], fold)
    assert not np.array_equal(0.0 + g.pairwise_sum(y2[:, :, 0]), np.sum(y2, axis=1)[:, 0])


@pytest.mark.parametrize('D', DIST_DIMS)
def test_statement_distance_equals_reference(D):
    import gauss_nd_double as g
    from elfi_b200.examples import gauss
    rs = np.random.RandomState(D)
    S = rs.randn(300, D) * np.exp(rs.randn(300, D) * 3)
    obs = rs.randn(1, D)
    S[0, 0], S[1, D - 1], S[2] = np.nan, np.inf, obs[0]
    with np.errstate(invalid='ignore'):
        want = gauss.euclidean_multidim(S, observed=[obs])
        assert same_bits(g.distance(S, obs[0]), want)
    seq = np.zeros(300)
    for j in range(D):
        seq = seq + (S[:, j] - obs[0, j]) ** 2
    with np.errstate(invalid='ignore'):
        differs = not np.array_equal(np.sqrt(seq)[3:], want[3:])
    assert differs == (D >= 8) or D == 8, D   # pairwise from D = 8 on (D = 8 may coincide)


# ---------------------------------------------------------------------------- the replay
def test_replay_numbers_the_normals_across_observations():
    """Normal q = t D + k of a row: the (n, D) normals are the n D normals of one row, in order."""
    import gauss_nd_replay as r
    for D in (1, 2, 3, 7, 16):
        z, _ = r.normals(5, 7, D, seed=11, offset=2 ** 32 - 2)
        flat, _ = r.normals(5, 7 * D, 1, seed=11, offset=2 ** 32 - 2)
        assert np.array_equal(z.reshape(5, -1), flat.reshape(5, -1)), D
        part, _ = r.normals(2, 7, D, seed=11, offset=2 ** 32 + 1)
        assert np.array_equal(part, z[3:]), D


def test_replay_law():
    """The replayed rows have means mu and covariance A^T A = cov."""
    import gauss_nd_replay as r
    from elfi_b200 import ops
    cov = np.array([[1.0, .5, 0.0], [.5, 1.0, -.3], [0.0, -.3, 2.0]])
    A = ops.gauss_nd_factor(cov, 3)
    assert np.allclose(A.T @ A, cov)
    mu = np.array([[1.0, -2.0, 3.0]])
    Y, err = r.sim_gauss_nd(mu, A, 100000, seed=3)
    x = Y[0]
    assert np.all(np.abs(x.mean(axis=0) - mu[0]) < 5 * np.sqrt(np.diag(cov) / 1e5))
    assert np.allclose(np.cov(x, rowvar=False), cov, atol=0.03)
    assert np.all(err < 1e-12 * (1 + np.abs(Y)))


def test_factor_follows_numpy_and_scipy():
    from elfi_b200 import ops
    for cov, D in (([1], 1), (None, 4), (2.0, 3), ([[1, .5], [.5, 1]], 2),
                   ([[1, 1], [1, 1]], 2)):
        A = ops.gauss_nd_factor(cov, D)
        c = np.asarray(1.0 if cov is None else cov, dtype=float)
        c = c * np.eye(D) if c.ndim == 0 else (np.diag(c) if c.ndim == 1 else c)
        _, s, vh = np.linalg.svd(c)
        assert np.array_equal(A, np.sqrt(s)[:, None] * vh)
    with pytest.raises(ValueError, match='positive semidefinite'):
        ops.gauss_nd_factor([[1, 2], [2, 1]], 2)
    with pytest.raises(ValueError, match=r'\(3, 3\)'):
        ops.gauss_nd_factor([[1, 0], [0, 1]], 3)


# ---------------------------------------------------------------------------- Python layer
@pytest.fixture
def nd_double(cpu_double, monkeypatch):
    import abi_double
    import gauss_nd_double
    import priors_double
    abi_double.install(monkeypatch, priors_double.TABLE, gauss_nd_double.TABLE)
    return cpu_double


def _host(x):
    from elfi_b200 import device as dev
    return np.asarray(dev.to_host(x))


def _model(tag):
    from elfi_b200.examples import gauss
    tp, cov = CONFIGS[tag]
    return gauss.get_model(true_params=tp, seed_obs=SEED_OBS[tag], nd_mean=True, cov_matrix=cov)


@pytest.mark.parametrize('tag', sorted(CONFIGS))
def test_observed_and_generate_match_reference_golden(nd_double, tag):
    g = load_golden('gauss_nd')
    m = _model(tag)
    D = len(CONFIGS[tag][0])
    assert m.parameter_names == ['mu_{}'.format(i) for i in range(D)]
    assert same_bits(m.observed['gauss'], g[tag + '_observed'])
    out = m.generate(20, seed=11)
    for k in ['mu_{}'.format(i) for i in range(D)] + ['gauss', 'ss_mean', 'ss_var', 'd']:
        assert same_bits(_host(out[k]), g['{}_gen_{}'.format(tag, k)]), k


@pytest.mark.parametrize('tag', sorted(CONFIGS))
@pytest.mark.parametrize('run', sorted(REJECTION))
def test_rejection_matches_reference_golden(nd_double, tag, run):
    import elfi_b200 as elfi
    g = load_golden('gauss_nd')
    init, kw = REJECTION[run]
    if run == 'threshold':
        kw = dict(kw, threshold=THRESHOLD[tag])
    res = elfi.Rejection(_model(tag)['d'], **init).sample(bar=False, **kw)
    pre = '{}_{}_'.format(tag, run)
    assert res.n_sim == int(g[pre + 'n_sim'])
    assert res.threshold == float(g[pre + 'threshold'])
    assert same_bits(res.discrepancies, g[pre + 'd'])
    for i in range(len(CONFIGS[tag][0])):
        assert same_bits(res.samples['mu_{}'.format(i)], g[pre + 'mu_{}'.format(i)]), i


@pytest.mark.parametrize('tag', sorted(CONFIGS))
def test_smc_matches_reference_golden(nd_double, tag):
    import elfi_b200 as elfi
    g = load_golden('gauss_nd')
    res = elfi.SMC(_model(tag)['d'], batch_size=1000, seed=20).sample(
        150, thresholds=SMC_THRESHOLDS[tag], bar=False)
    pre = tag + '_smc_'
    names = ['mu_{}'.format(i) for i in range(len(CONFIGS[tag][0]))]
    assert res.n_sim == int(g[pre + 'n_sim'])
    assert len(res.populations) == int(g[pre + 'n_pops'])
    for i, pop in enumerate(res.populations):
        p = '{}pop{}_'.format(pre, i)
        assert pop.n_sim == int(g[p + 'n_sim']), i
        got = dict({k: pop.samples[k] for k in names}, d=pop.discrepancies)
        for k, v in got.items():
            if i == 0:
                assert same_bits(v, g[p + k]), (i, k)
            else:
                np.testing.assert_allclose(v, g[p + k], rtol=RTOL, atol=ATOL, err_msg=str((i, k)))
        np.testing.assert_allclose(pop.weights, g[p + 'weights'], rtol=1e-5)
    np.testing.assert_allclose(res.discrepancies, g[pre + 'd'], rtol=RTOL, atol=ATOL)
    np.testing.assert_allclose(res.threshold, float(g[pre + 'threshold']), rtol=1e-7)


def test_one_d_model_is_unchanged(nd_double):
    from elfi_b200.examples import gauss
    m = gauss.get_model(seed_obs=2)
    assert m.parameter_names == ['mu', 'sigma']
    assert m.observed['gauss'].shape == (1, 50)
    out = m.generate(10, seed=1)
    assert _host(out['ss_mean']).shape == (10,) and _host(out['d']).shape == (10,)


def test_reference_gauss_1d_and_2d_mean(nd_double):
    """The reference's test_gauss_1d_mean and test_gauss_2d_mean (tests/unit/test_examples.py)."""
    import elfi_b200 as elfi
    from elfi_b200.examples import gauss
    for params_true, cov_matrix in (([4], [1]), ([4, 4], [[1, .5], [.5, 1]])):
        m = gauss.get_model(true_params=params_true, nd_mean=True, cov_matrix=cov_matrix)
        res = elfi.Rejection(m, m['d'], batch_size=10).sample(20, bar=False)
        assert len(res.samples['mu_0']) == 20


def test_ops_validate_before_the_call(nd_double):
    import abi_double
    from elfi_b200 import ops
    del abi_double.CALLS[:]
    A = np.eye(2)
    with pytest.raises(ValueError, match=r'1 <= D <= 16.*\(4, 17\)'):
        ops.sim_gauss_nd(np.zeros((4, 17)), np.eye(17))
    with pytest.raises(ValueError, match='n_obs <= 7688, got 7689'):
        ops.sim_gauss_nd(np.zeros((4, 2)), A, n_obs=7689)
    with pytest.raises(ValueError, match='n_obs <= 7688, got 0'):
        ops.sim_gauss_nd(np.zeros((4, 2)), A, n_obs=0)
    with pytest.raises(ValueError, match=r'\(2, 2\), got shape \(3, 3\)'):
        ops.sim_gauss_nd(np.zeros((4, 2)), np.eye(3))
    with pytest.raises(ValueError, match='one length'):
        ops.sim_gauss_nd([np.zeros(3), np.zeros(4)], A)
    with pytest.raises(ValueError, match='neither'):
        ops.sim_gauss_nd(np.zeros((4, 2)), A, want_summaries=False)
    with pytest.raises(ValueError, match=r'\(batch, n, D\) data, got shape \(4, 5\)'):
        ops.gauss_nd_summaries(np.zeros((4, 5)))
    with pytest.raises(ValueError, match=r'1 <= n .* got shape \(4, 0, 2\)'):
        ops.gauss_nd_summaries(np.zeros((4, 0, 2)))
    with pytest.raises(ValueError, match=r'\(batch, D\) data, got shape \(4,\)'):
        ops.gauss_nd_distance(np.zeros(4), np.zeros(1))
    with pytest.raises(ValueError, match='same number of columns'):
        ops.gauss_nd_distance(np.zeros((4, 3)), np.zeros(2))
    assert abi_double.CALLS == []


def test_device_model_dispatch(nd_double):
    """The device model: a lazy (B, n_obs, D) output whose fused summaries equal the summary entry
    point of its materialised data; ss_mean / ss_var of rank-3 lazy, host and device data; the
    distance on the device; and the arguments it refuses."""
    import abi_double
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    from elfi_b200.examples import gauss
    from elfi_b200.throughput import LazySimulation
    cov = [[1, .5], [.5, 1]]
    m, dp = gauss.get_device_model(n_obs=15, nd_mean=True, cov_matrix=cov, seed_obs=1)
    assert dp.parameter_names == ['mu_0', 'mu_1']
    assert same_bits(m.observed['gauss'], gauss.get_model(n_obs=15, nd_mean=True, cov_matrix=cov,
                                                          seed_obs=1).observed['gauss'])
    A = ops.gauss_nd_factor(cov, 2)
    y = gauss.gauss_nd_device(np.arange(5.0), np.ones(5), A=A, n_obs=15, batch_size=5,
                              random_state=np.random.RandomState(0))
    assert isinstance(y, LazySimulation) and y.shape == (5, 15, 2)
    del abi_double.CALLS[:]
    mean, var = gauss.ss_mean(y), gauss.ss_var(y)
    assert abi_double.CALLS == ['elfi_b200_sim_gauss_nd_f64']
    data = y.materialize()
    assert data is y.materialize() and tuple(data.shape) == (5, 15, 2)
    S = ops.gauss_nd_summaries(data)
    assert same_bits(_host(mean), _host(S)[:, :2]) and same_bits(_host(var), _host(S)[:, 2:])
    assert same_bits(_host(gauss.ss_mean(_host(data))), _host(mean))
    assert same_bits(_host(gauss.ss_var(data)), _host(var))
    obs = gauss.ss_mean(m.observed['gauss'])
    d = gauss.euclidean_multidim(mean, var, observed=[obs, None])
    assert dev.is_device_array(d)
    import gauss_nd_double as g
    assert same_bits(_host(d), g.distance(_host(mean), _host(obs)[0]))
    out = m.generate(64, seed=3)
    assert _host(out['d']).shape == (64,)
    with pytest.raises(ValueError, match='1 <= D <= 16 means, got 17'):
        gauss.get_device_model(nd_mean=True, true_params=[4] * 17)
    with pytest.raises(ValueError, match='n_obs <= 7688'):
        gauss.get_device_model(nd_mean=True, n_obs=10 ** 4)
