"""CPU checks of the M/G/1 example.

* the host path of elfi_b200.examples.mg1 against the golden fixtures of the unmodified reference
  (tests/golden/gen_golden_mg1.py), bit for bit: draws, summaries, the conditional prior's
  ModelPrior density and a Rejection sample; the graph names match the reference;
* elfi_b200/csrc/mg1.cuh built for the host (tests/harness/mg1_harness.cpp): the recurrence fed the
  W and U the reference draws equals its arithmetic (NaN and inf included), the draws from
  uniforms equal NumPy's formulas, and the pick / lerp path equals np.quantile on sorted rows for
  every n in 2..512;
* the Python layer (validation, dispatch, the throughput-mode graph) and the samplers on the CPU
  test double extended by tests/mg1_double.py.
"""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import load_golden

HERE = os.path.dirname(os.path.abspath(__file__))
Q10 = np.linspace(0, 1, 10)


@pytest.fixture(scope='module')
def harness(tmp_path_factory):
    gxx = shutil.which('g++')
    if gxx is None:
        pytest.skip('g++ not available')
    so = str(tmp_path_factory.mktemp('mg1') / 'mg1_harness.so')
    subprocess.check_call([gxx, '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-o', so,
                           os.path.join(HERE, 'harness', 'mg1_harness.cpp')])
    return ctypes.CDLL(so)


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _same_bits(a, b):
    """Equal values, NaN where NaN, and the same sign of every zero."""
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True) and \
        np.array_equal(np.signbit(a[a == 0]), np.signbit(b[a == 0]))


class _GivenDraws:
    """A RandomState stand-in that hands out given W and U in the order they are asked for."""

    def __init__(self, W, U):
        self.W, self.U = W, U

    def exponential(self, scale, size):
        return np.broadcast_to(scale, size[1:]) * self.W

    def uniform(self, low, high, size):
        return low + (np.broadcast_to(high, size[1:]) - low) * self.U


# ---------------------------------------------------------------------------- reference goldens
def test_host_draws_match_reference_golden():
    from elfi_b200.examples import mg1
    g = load_golden('mg1_draws')
    assert np.array_equal(mg1.MG1(1., 5., 0.2, batch_size=1, random_state=np.random.RandomState(1)),
                          g['y1'])
    prm = g['prm']
    yb = mg1.MG1(prm[:, 0], prm[:, 1], prm[:, 2], batch_size=len(prm),
                 random_state=np.random.RandomState(2))
    assert np.array_equal(yb, g['yb'])
    ys = mg1.MG1(prm[:, 0], prm[:, 1], prm[:, 2], n_obs=7, batch_size=len(prm),
                 random_state=np.random.RandomState(3))
    assert np.array_equal(ys, g['ys'])


def test_host_summaries_match_reference_golden():
    from elfi_b200.examples import mg1
    g = load_golden('mg1_summaries')
    d = load_golden('mg1_draws')
    with np.errstate(all='ignore'):
        for name in ('y1', 'yb', 'ys'):
            assert _same_bits(mg1.log_identity(d[name]), g[name + '_log']), name
            assert _same_bits(mg1.quantiles(d[name], Q10), g[name + '_q10']), name
        for name in ('crafted', 'n2'):
            assert _same_bits(mg1.quantiles(g[name], Q10), g[name + '_q10']), name
            assert _same_bits(mg1.quantiles(g[name], g['qr']), g[name + '_qr']), name


def test_prior_logpdf_matches_reference_golden(cpu_double):
    import elfi_b200 as elfi
    from elfi_b200.examples import mg1
    g = load_golden('mg1_prior_logpdf')
    m = mg1.get_model(seed_obs=1)
    assert m.parameter_names == list(g['names'])
    with np.errstate(all='ignore'):
        lp = elfi.ModelPrior(m).logpdf(g['x'])
    assert _same_bits(lp, g['logpdf'])
    assert np.isneginf(g['logpdf']).sum() >= 8 and np.isfinite(g['logpdf']).sum() >= 10


def test_rejection_matches_reference_golden(cpu_double):
    import elfi_b200 as elfi
    from elfi_b200.examples import mg1
    g = load_golden('mg1_rejection')
    m = mg1.get_model(seed_obs=1)
    assert np.array_equal(m.observed['MG1'], g['observed'])
    res = elfi.Rejection(m['d'], batch_size=100, seed=3).sample(20, quantile=0.1, bar=False)
    assert res.n_sim == int(g['n_sim'])
    assert res.threshold == float(g['threshold'])
    assert np.array_equal(res.discrepancies, g['d'])
    for name in ('t1', 't2', 't3'):
        assert np.array_equal(res.samples[name], g['out_' + name]), name


def test_graph_names_match_the_reference():
    from elfi_b200.examples import mg1
    m = mg1.get_model(seed_obs=0, n_quantiles=5)
    assert m.parameter_names == ['t1', 't2', 't3']
    assert {'t1', 't2', 't3', 'MG1', 'log_identity', 'quantiles', 'd'} <= set(m.nodes)
    assert m.get_parents('t2')[0] == 't1'


# ---------------------------------------------------------------------------- mg1.cuh on the host
def test_recurrence_equals_the_reference_arithmetic(harness):
    """The header's step, fed the W and U the reference draws, gives its series bit for bit, NaN
    and inf included; the rows where the reference raises are NaN."""
    from elfi_b200.examples import mg1
    rs = np.random.RandomState(7)
    B, n = 300, 50
    t1 = rs.uniform(0, 10, B)
    P = np.column_stack([t1, t1 + rs.uniform(0, 10, B), rs.uniform(0, 0.5, B)])
    P[:6] = [(1, 5, 0.2), (3, 3, 0.2), (0, 10, 1e-300), (1, 5, 0.0), (1, 5, np.nan), (0, 0, 0.5)]
    W = rs.exponential(1.0, (n, B))
    U = rs.uniform(0, 1, (n, B))
    W[5, 10], W[7, 11], U[3, 12], U[9, 13] = np.inf, np.nan, np.nan, np.inf
    W[:, 14] = 0.0
    with np.errstate(all='ignore'):
        want = mg1.MG1(P[:, 0], P[:, 1], P[:, 2], n_obs=n, batch_size=B,
                       random_state=_GivenDraws(W, U))
        Wr = (1 / P[:, 2]) * W
        Ur = P[:, 0] + (P[:, 1] - P[:, 0]) * U
    Y = np.empty((B, n))
    harness.harness_mg1_rows(_ptr(np.ascontiguousarray(P)), _ptr(np.ascontiguousarray(Wr.T)),
                             _ptr(np.ascontiguousarray(Ur.T)), ctypes.c_int64(B), ctypes.c_int32(n),
                             _ptr(Y))
    assert _same_bits(Y, want)
    assert np.isnan(Y).any() and np.isinf(Y).any()
    # the rows where NumPy raises come out NaN
    bad = np.array([(1, 5, -0.2), (1, 5, -0.0), (1, 5, -np.inf), (1, np.inf, 0.2),
                    (np.nan, 5, 0.2), (-np.inf, 5, 0.2)])
    for row in bad:
        with pytest.raises((ValueError, OverflowError)):
            with np.errstate(all='ignore'):
                mg1.MG1(*row, n_obs=3, random_state=np.random.RandomState(0))
    Yb = np.empty((len(bad), 4))
    Wb = np.ones((len(bad), 4))
    harness.harness_mg1_rows(_ptr(np.ascontiguousarray(bad)), _ptr(Wb), _ptr(Wb.copy()),
                             ctypes.c_int64(len(bad)), ctypes.c_int32(4), _ptr(Yb))
    assert np.isnan(Yb).all()


def test_draws_equal_numpy_formulas(harness):
    rs = np.random.RandomState(2)
    B, n = 50, 20
    P = np.column_stack([rs.uniform(0, 10, B), rs.uniform(0, 20, B), rs.uniform(0, 0.5, B)])
    P[:3, 2] = [0.0, np.nan, 1e-300]
    u, v = 1.0 - rs.random_sample((B, n)), 1.0 - rs.random_sample((B, n))
    u[0, 0] = 1.0
    W, U = np.empty((B, n)), np.empty((B, n))
    harness.harness_mg1_draws(_ptr(P), _ptr(u), _ptr(v), ctypes.c_int64(B), ctypes.c_int32(n),
                              _ptr(W), _ptr(U))
    with np.errstate(all='ignore'):
        assert _same_bits(U, P[:, :1] + (P[:, 1:2] - P[:, :1]) * v)
        want = (1 / P[:, 2:3]) * -np.log(u)
    assert np.array_equal(np.isnan(W), np.isnan(want))
    f = np.isfinite(want)
    np.testing.assert_allclose(W[f], want[f], rtol=4e-16)
    assert np.isinf(W[0, 1:]).all() and np.isnan(W[0, 0])


def test_quantile_picks_equal_numpy_for_every_n(harness):
    rs = np.random.RandomState(3)
    q = np.concatenate([Q10, rs.uniform(0, 1, 12), [0.5, 1 - 1e-17, 1e-300]])
    for n in range(2, 513):
        x = rs.exponential(1.0, (6, n)) * rs.uniform(1e-3, 1e3, (6, 1))
        x[1] = np.round(x[1])
        x[2, rs.randint(n)] = np.inf
        x[3, rs.randint(n)] = -np.inf
        x[4, rs.randint(n)] = np.nan
        x[5, :] = rs.choice([0.0, 1.0], n)          # ties (np.quantile's partition does not keep
        x[5, 0] = -0.0                                # the order of -0.0 and 0.0; a lone one is kept)
        xs = np.sort(x, axis=1)
        S = np.empty((6, q.size))
        harness.harness_mg1_quantiles(_ptr(np.ascontiguousarray(xs)), ctypes.c_int64(6),
                                      ctypes.c_int32(n), _ptr(q), ctypes.c_int32(q.size), _ptr(S))
        with np.errstate(all='ignore'):
            assert _same_bits(S, np.quantile(x, q, axis=1).T), n


# ---------------------------------------------------------------------------- Python layer
@pytest.fixture
def mg1_double(cpu_double, monkeypatch):
    import abi_double
    import mg1_double
    import priors_double
    abi_double.install(monkeypatch, priors_double.TABLE, mg1_double.TABLE)
    return cpu_double


def test_ops_validate_before_the_call(mg1_double):
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    with pytest.raises(ValueError, match='observations'):
        ops.sim_mg1(np.ones((2, 3)), n_obs=1)
    with pytest.raises(ValueError, match='observations'):
        ops.sim_mg1(np.ones((2, 3)), n_obs=513)
    with pytest.raises(ValueError, match='levels'):
        ops.sim_mg1(np.ones((2, 3)), q=np.linspace(0, 1, 33))
    with pytest.raises(ValueError, match='levels'):
        ops.sim_mg1(np.ones((2, 3)), q=[])
    with pytest.raises(ValueError, match=r'\[0, 1\]'):
        ops.sim_mg1(np.ones((2, 3)), q=[0.5, 1.5])
    with pytest.raises(ValueError, match='3 parameters'):
        ops.sim_mg1(np.ones((2, 2)))
    with pytest.raises(ValueError, match='observations'):
        ops.row_quantiles(dev.to_device(np.ones((2, 1))), Q10)
    with pytest.raises(ValueError, match='observations'):
        ops.row_quantiles(dev.to_device(np.ones((2, 513))), Q10)
    with pytest.raises(ValueError, match=r'\[0, 1\]'):
        ops.row_quantiles(dev.to_device(np.ones((2, 5))), [-0.1])
    with pytest.raises(ValueError, match='batch, n'):
        ops.row_quantiles(dev.to_device(np.ones((2, 3, 4))), Q10)
    assert not mg1_double.CALLS


def test_dispatch_host_device_and_lazy_agree(mg1_double):
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    from elfi_b200.examples import mg1
    rs = np.random.RandomState(0)
    full = rs.exponential(1.0, (6, 41))
    full[0, 3] = np.nan
    y = full[:, 1:]
    for src in (dev.to_device(y), dev.to_device(full)[:, 1:]):
        assert _same_bits(mg1.quantiles(src, Q10).cpu().numpy(), mg1.quantiles(y, Q10))
        got = mg1.log_identity(src).cpu().numpy()
        np.testing.assert_allclose(got, np.log(y), rtol=1e-15)
    lazy = mg1.mg1_device(1., 5., 0.2, n_obs=30, batch_size=5, random_state=np.random.RandomState(1))
    data = lazy.materialize()
    assert tuple(data.shape) == (5, 30) and lazy.shape == (5, 30)
    assert _same_bits(mg1.quantiles(lazy, Q10).cpu().numpy(), mg1.quantiles(data.cpu().numpy(), Q10))
    q3 = [0.1, 0.5, 0.9]
    assert _same_bits(mg1.quantiles(lazy, q3).cpu().numpy(), mg1.quantiles(data.cpu().numpy(), q3))
    np.testing.assert_allclose(mg1.log_identity(lazy).cpu().numpy(), np.log(data.cpu().numpy()),
                               rtol=1e-15)
    Y, S = ops.sim_mg1(np.tile([1., 5., 0.2], (4, 1)), n_obs=20, q=q3, want_data=True)
    assert _same_bits(S.cpu().numpy(), np.quantile(Y.cpu().numpy(), q3, axis=1).T)
    Y, _ = ops.sim_mg1([[1., 5., -0.0], [1., np.inf, 0.2], [1., 5., 0.2]], n_obs=5, want_data=True)
    Y = Y.cpu().numpy()
    assert np.isnan(Y[:2]).all() and np.isfinite(Y[2]).all()


def test_device_model_runs_rejection_and_smc(mg1_double):
    import elfi_b200 as elfi
    from elfi_b200.examples import mg1
    m, dp = mg1.get_device_model(seed_obs=3)
    assert dp.parameter_names == ['t1', 't2', 't3']
    np.testing.assert_array_equal(dp.sources, [[-1, -1], [0, -1], [-1, -1]])
    host = mg1.get_model(seed_obs=3)
    assert np.array_equal(m.observed['MG1'], host.observed['MG1'])

    def in_support(s):
        return np.all((s['t2'] >= s['t1']) & (s['t2'] <= s['t1'] + 10) & (s['t1'] >= 0) &
                      (s['t1'] <= 10) & (s['t3'] >= 0) & (s['t3'] <= 0.5))
    res = elfi.Rejection(m['d'], batch_size=500, seed=1).sample(50, quantile=0.1, bar=False)
    assert res.n_samples == 50 and in_support(res.samples)
    smc = elfi.SMC(m['d'], batch_size=500, seed=2, device_proposal=dp).sample(
        50, quantiles=[0.5, 0.5], bar=False)
    assert len(smc.populations) == 2 and in_support(smc.samples)
    m['d'].become(elfi.AdaptiveDistance(m['quantiles']))
    ad = elfi.AdaptiveDistanceSMC(m['d'], batch_size=500, seed=3, device_proposal=dp).sample(
        50, rounds=2, quantile=0.5, bar=False)
    assert len(ad.populations) == 2 and in_support(ad.samples)
    for name in ('elfi_b200_sim_mg1_f64', 'elfi_b200_prior_rvs_cond_f64',
                 'elfi_b200_prior_logpdf_cond_f64', 'elfi_b200_gm_rvs_cdf_f64'):
        assert name in mg1_double.CALLS, name
    with pytest.raises(ValueError, match='observations'):
        mg1.get_device_model(n_obs=600)
