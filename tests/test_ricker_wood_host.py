"""CPU checks of Wood's 13 Ricker statistics (ss_wood of elfi_b200.examples.ricker):

* the host definition against the row-by-row restatement of tests/ricker_wood_cases.py on host
  Ricker draws, at the truth and at prior draws, and bit for bit against np.mean / np.var;
* the rank rule of the autoregression on degenerate rows, non-finite rows, the observed series'
  own cubic coefficients;
* the Python layer (the summary='wood' graphs, argument checks, dispatch to the kernel for device
  data and lazy simulator output) and a BSL run, on the CPU test doubles.
"""
import numpy as np
import pytest
import scipy.stats as ss

import ricker_wood_cases as rwc

TRUTH = (3.8, 0.3, 10.0)


def _draws(n_obs, seed, B=40):
    """Host Ricker series: B // 2 rows at the truth, B // 2 at prior draws (extinctions, bursts)."""
    from elfi_b200.examples import ricker
    rs = np.random.RandomState(seed)
    truth = ricker.stochastic_ricker(*TRUTH, n_obs=n_obs, batch_size=B // 2, random_state=rs)
    prm = np.column_stack([ss.expon.rvs(np.e, 2, size=B // 2, random_state=rs),
                           ss.truncnorm.rvs(0, 5, size=B // 2, random_state=rs),
                           rs.uniform(0, 100, B // 2)])
    prior = np.array([ricker.stochastic_ricker(*p, n_obs=n_obs, random_state=rs)[0] for p in prm])
    obs = ricker.stochastic_ricker(*TRUTH, n_obs=n_obs, random_state=rs)
    return np.concatenate([truth, prior]), obs


@pytest.mark.parametrize('n_obs', [7, 50, 129, 500])
def test_host_definition_matches_restatement(n_obs):
    from elfi_b200.examples import ricker
    y, obs = _draws(n_obs, n_obs)
    S = ricker.ss_wood(y, obs)
    assert S.shape == (len(y), 13)
    np.testing.assert_array_equal(S[:, 0], np.mean(y, axis=1))
    np.testing.assert_array_equal(S[:, 2], np.var(y, axis=1))
    P = rwc.design(obs)
    np.testing.assert_array_equal(ricker.wood_design(obs), P)
    rwc.check(S, rwc.restate_rows(y, P), y, P, exact_sums=False)
    kinds = {rwc.rank_kind(r) for r in y}
    assert 'full' in kinds


def test_rank_rule_on_degenerate_rows():
    from elfi_b200.examples import ricker
    n = 12
    rs = np.random.RandomState(1)
    zeros = np.zeros(n)
    ones = (rs.uniform(size=n) < 0.5).astype(float)
    ones[[0, 1]] = [1.0, 1.0]
    sevens = 7.0 * (rs.uniform(size=n) < 0.5)
    sevens[[2, 3]] = [7.0, 0.0]
    y = np.array([zeros, ones, sevens])
    obs = rs.poisson(5.0, n).astype(float)
    S = ricker.ss_wood(y, obs)
    assert S[0, 1] == n and np.all(np.delete(S[0], 1) == 0)
    for row, k in ((ones, 1.0), (sevens, 7.0)):
        assert rwc.rank_kind(row) == 'one'
    for i, k in ((1, 1.0), (2, 7.0)):
        at_k = y[i, :-1] == k
        s = np.mean(y[i, 1:][at_k] ** 0.3)
        den = k ** 0.6 + k ** 1.2
        np.testing.assert_allclose(S[i, 11:], [s * k ** 0.3 / den, s * k ** 0.6 / den], rtol=4 * rwc.U)
    np.testing.assert_allclose(S[1, 11], S[1, 12], rtol=0)      # k = 1: proportional, equal
    rwc.check(S, rwc.restate_rows(y, rwc.design(obs)), y, rwc.design(obs), exact_sums=False)


def test_non_finite_rows_give_nan():
    from elfi_b200.examples import ricker
    rs = np.random.RandomState(2)
    y = rs.poisson(8.0, (4, 20)).astype(float)
    y[1, 5], y[2, 19], y[3, 0] = np.nan, np.inf, -np.inf
    S = ricker.ss_wood(y, rs.poisson(8.0, 20).astype(float))
    assert np.all(np.isfinite(S[0])) and np.isnan(S[1:]).all()


@pytest.mark.parametrize('n_obs', [50, 129, 500])
def test_observed_series_cubic_coefficients_are_identity(n_obs):
    from elfi_b200.examples import ricker
    obs = ricker.stochastic_ricker(*TRUTH, n_obs=n_obs, random_state=np.random.RandomState(n_obs))
    o = np.sort(np.diff(obs[0]))
    assert np.linalg.matrix_rank(np.column_stack([o, o ** 2, o ** 3])) == 3
    c = ricker.ss_wood(obs, obs)[0, 8:11]
    assert np.all(np.abs(c - [1.0, 0.0, 0.0]) < 1e-10), c


def test_get_model_wood_node_and_argument_errors():
    from elfi_b200 import model as em
    from elfi_b200.examples import ricker
    m = ricker.get_model(seed_obs=3, summary='wood')
    assert isinstance(m['Wood'], em.Summary) and 'd' not in m.nodes and 'Mean' not in m.nodes
    out = m.generate(25, ['Wood', 'Ricker'], seed=4)
    assert out['Wood'].shape == (25, 13)
    np.testing.assert_array_equal(out['Wood'], ricker.ss_wood(out['Ricker'], m.observed['Ricker']))
    assert np.shape(m['Wood'].observed) == (1, 13)
    default = ricker.get_model(seed_obs=3)
    assert {'Mean', 'Var', '#0', 'd'} <= set(default.nodes) and 'Wood' not in default.nodes
    with pytest.raises(ValueError, match='stochastic'):
        ricker.get_model(stochastic=False, summary='wood')
    with pytest.raises(ValueError, match='summary'):
        ricker.get_model(summary='nope')
    with pytest.raises(ValueError, match='n_obs'):
        ricker.get_model(n_obs=6, summary='wood')
    with pytest.raises(ValueError, match='n_obs'):
        ricker.ss_wood(np.zeros((2, 6)), np.zeros(6))
    with pytest.raises(ValueError, match='observed series'):
        ricker.ss_wood(np.zeros((2, 10)), np.zeros(11))
    with pytest.raises(ValueError, match='one row'):
        ricker.ss_wood(np.zeros((2, 10)), np.zeros((2, 10)))


# ---------------------------------------------------------------------------- Python layer
@pytest.fixture
def wood_double(cpu_double, monkeypatch):
    import abi_double
    abi_double.install(monkeypatch, *_wood_tables())
    return cpu_double


def _wood_tables():
    import priors_double
    import ricker_double
    import ricker_wood_double
    return priors_double.TABLE, ricker_double.TABLE, ricker_wood_double.TABLE


def test_device_model_arguments(wood_double):
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    from elfi_b200.examples import ricker
    with pytest.raises(ValueError, match='stochastic'):
        ricker.get_device_model(stochastic=False, summary='wood')
    with pytest.raises(ValueError, match='summary'):
        ricker.get_device_model(summary='Wood')
    for n_obs in (6, ops.RICKER_WOOD_NOBS_MAX + 1):
        with pytest.raises(ValueError, match='n_obs'):
            ricker.get_device_model(n_obs=n_obs, summary='wood')
    y = dev.to_device(np.ones((3, 10)))
    with pytest.raises(ValueError, match=r'\(3, 9\)'):
        ops.wood_summaries(y, np.ones((3, 10)))
    with pytest.raises(ValueError, match='n_obs'):
        ops.wood_summaries(dev.to_device(np.ones((3, 6))), np.ones((3, 5)))
    assert 'elfi_b200_ricker_wood_f64' not in wood_double.CALLS


def test_dispatch_host_device_and_lazy_agree(wood_double):
    from elfi_b200 import device as dev
    from elfi_b200.examples import ricker
    y, obs = _draws(30, 5)
    host = ricker.ss_wood(y, obs)
    np.testing.assert_array_equal(ricker.ss_wood(dev.to_device(y), obs).cpu().numpy(), host)
    wide = dev.to_device(np.concatenate([y, np.ones((len(y), 4))], axis=1))[:, :30]
    np.testing.assert_array_equal(ricker.ss_wood(wide, obs).cpu().numpy(), host)
    assert ricker._wood_design(obs, 30, True) is ricker._wood_design(obs, 30, True)
    lazy = ricker.ricker_device(*TRUTH, n_obs=30, batch_size=6, random_state=np.random.RandomState(2))
    data = lazy.materialize().cpu().numpy()
    np.testing.assert_array_equal(ricker.ss_wood(lazy, obs).cpu().numpy(), ricker.ss_wood(data, obs))
    assert 'elfi_b200_ricker_wood_f64' in wood_double.CALLS
    m, dp = ricker.get_device_model(seed_obs=3, summary='wood')
    assert dp.parameter_names == ['t1', 't2', 't3'] and 'd' not in m.nodes
    out = m.generate(20, ['Wood', 'Ricker'], seed=1)
    assert tuple(out['Wood'].shape) == (20, 13)
    np.testing.assert_array_equal(
        out['Wood'].cpu().numpy(),
        ricker.ss_wood(out['Ricker'].materialize().cpu().numpy(), m.observed['Ricker']))


def test_bsl_on_the_host_model(wood_double, monkeypatch):
    import abi_double
    import bsl_double
    from elfi_b200 import bsl
    from elfi_b200.examples import ricker
    abi_double.install(monkeypatch, *_wood_tables(), bsl_double.TABLE)
    m = ricker.get_model(seed_obs=4, summary='wood')
    # the statistics' variances span ~16 orders of magnitude, beyond the likelihood's pivot cut
    # (relative to the largest variance): without a common scale every round gives -inf
    pilot = m.generate(1000, ['Wood'], with_values=dict(zip(['t1', 't2', 't3'], TRUTH)),
                       seed=2)['Wood']
    with pytest.raises(RuntimeError, match='not finite'):
        bsl.BSL(m, 200, ['Wood'], seed=7).sample(2, np.diag([0.01, 0.001, 0.5]),
                                                 params0=np.array(TRUTH))
    lik = bsl.standard_likelihood(whitening=np.diag(1 / np.std(pilot, axis=0)))
    sampler = bsl.BSL(m, 200, ['Wood'], likelihood=lik, seed=7)
    res = sampler.sample(20, np.diag([0.01, 0.001, 0.5]), params0=np.array(TRUTH))
    assert sampler.observed.shape == (1, 13)
    assert np.all(np.isfinite(sampler.state['logposterior']))
    assert res.n_sim == 20 * 200
