"""CPU checks of the ARCH(1) example.

* the host path of elfi_b200.examples.arch against the golden fixtures of the unmodified reference
  (tests/golden/gen_golden_arch.py), bit for bit: draws, summaries, Rejection, and the n_obs quirk
  (observed series of get_model's n_obs, simulated ones of 100);
* elfi_b200/csrc/arch.cuh built for the host (tests/harness/arch_harness.cpp): the recurrence fed
  the same normals as the reference's arithmetic, and the summaries against NumPy at every n in
  2..128 and every n_lags in 1..8, NaN, inf and signed zeros included;
* the Python layer (validation, dispatch, the throughput-mode graph) and the samplers on the CPU
  test double extended by tests/arch_double.py.
"""
import ctypes
import os
import shutil
import subprocess
from itertools import combinations

import numpy as np
import pytest

from conftest import load_golden

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope='module')
def harness(tmp_path_factory):
    gxx = shutil.which('g++')
    if gxx is None:
        pytest.skip('g++ not available')
    so = str(tmp_path_factory.mktemp('arch') / 'arch_harness.so')
    subprocess.check_call([gxx, '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-o', so,
                           os.path.join(HERE, 'harness', 'arch_harness.cpp')])
    return ctypes.CDLL(so)


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _rows(harness, P, z):
    P = np.ascontiguousarray(P, dtype=np.float64)
    z = np.ascontiguousarray(z, dtype=np.float64)
    B, n = z.shape[0], z.shape[1] - 1
    Y = np.empty((B, n))
    harness.harness_arch_rows(_ptr(P), _ptr(z), ctypes.c_int64(B), ctypes.c_int32(n), _ptr(Y))
    return Y


def _summaries(harness, x, n_lags):
    x = np.ascontiguousarray(x, dtype=np.float64)
    S = np.empty((x.shape[0], 2 + n_lags + n_lags * (n_lags - 1) // 2))
    harness.harness_arch_summaries(_ptr(x), ctypes.c_int64(x.shape[0]), ctypes.c_int32(x.shape[1]),
                                   ctypes.c_int32(n_lags), _ptr(S))
    return S


def _reference_summaries(x, n_lags):
    from elfi_b200.examples import arch
    with np.errstate(all='ignore'):
        cols = [arch.sample_mean(x), arch.sample_variance(x)]
        cols += [arch.autocorr(x, i) for i in range(1, n_lags + 1)]
        cols += [arch.pairwise_autocorr(x, i, j) for i, j in combinations(range(1, n_lags + 1), 2)]
    return np.column_stack(cols)


def _same_bits(a, b):
    """Equal values, NaN where NaN, and the same sign of every zero."""
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True) and \
        np.array_equal(np.signbit(a[a == 0]), np.signbit(b[a == 0]))


class _GivenNormals:
    """A RandomState stand-in that hands out given arrays in the order they are asked for."""

    def __init__(self, *arrays):
        self.arrays = list(arrays)

    def normal(self, size):
        a = self.arrays.pop(0)
        assert a.shape == (size if isinstance(size, tuple) else (size,))
        return a


# ---------------------------------------------------------------------------- reference goldens
def test_host_draws_match_reference_golden():
    from elfi_b200.examples import arch
    g = load_golden('arch_draws')
    y1 = arch.arch(0.3, 0.7, batch_size=1, random_state=np.random.RandomState(1))
    assert np.array_equal(y1, g['y1'])
    prm = g['prm']
    yb = arch.arch(prm[:, 0], prm[:, 1], batch_size=len(prm), random_state=np.random.RandomState(2))
    assert np.array_equal(yb, g['yb'])
    ys = arch.arch(prm[:, 0], prm[:, 1], n_obs=17, batch_size=len(prm),
                   random_state=np.random.RandomState(3))
    assert np.array_equal(ys, g['ys'])


def test_host_summaries_match_reference_golden():
    g = load_golden('arch_summaries')
    draws = load_golden('arch_draws')
    data = dict(y1=draws['y1'], yb=draws['yb'], ys=draws['ys'], crafted=g['crafted'], n2=g['n2'],
                n128=g['n128'])
    keys = [k for k in g if '_L' in k]
    assert len(keys) == 11
    for key in keys:
        name, L = key.rsplit('_L', 1)
        assert _same_bits(_reference_summaries(data[name], int(L)), g[key]), key
    assert np.isnan(g['crafted_L5'][0, 2:]).all() and g['crafted_L5'][0, 1] == 0.0


def test_rejection_matches_reference_golden(cpu_double):
    """Rejection on get_model (host simulator and summaries) reproduces the reference's sample."""
    import elfi_b200 as elfi
    from elfi_b200.examples import arch
    g = load_golden('arch_rejection')
    m = arch.get_model(seed_obs=1)
    assert np.array_equal(m.observed['Y'], g['observed'])
    res = elfi.Rejection(m['d'], batch_size=100, seed=3).sample(20, quantile=0.1, bar=False)
    assert res.n_sim == int(g['n_sim'])
    assert res.threshold == float(g['threshold'])
    assert np.array_equal(res.discrepancies, g['d'])
    for name in ('t1', 't2'):
        assert np.array_equal(res.samples[name], g['out_' + name]), name


def test_n_obs_quirk_matches_reference_golden(cpu_double):
    """get_model(n_obs=40): the observed series has 40 observations, the simulator draws 100."""
    from elfi_b200 import device as dev
    from elfi_b200.examples import arch
    g = load_golden('arch_rejection')
    m = arch.get_model(n_obs=40, seed_obs=2)
    assert m.observed['Y'].shape == (1, 40)
    assert np.array_equal(m.observed['Y'], g['quirk_observed'])
    gen = m.generate(4, outputs=['t1', 't2', 'Y', 'd'], seed=5)
    assert gen['Y'].shape == (4, 100)
    for key in ('t1', 't2', 'Y', 'd'):
        v = dev.to_host(gen[key]) if dev.is_device_array(gen[key]) else gen[key]
        assert np.array_equal(np.asarray(v), g['quirk_' + key]), key


def test_graph_names_match_the_reference():
    from elfi_b200.examples import arch
    m = arch.get_model(seed_obs=0, n_lags=3)
    assert m.parameter_names == ['t1', 't2']
    names = set(m.nodes)
    assert {'t1', 't2', 'Y', 'MU', 'VAR', 'AC_1', 'AC_2', 'AC_3', 'PW_1_2', 'PW_1_3', 'PW_2_3',
            'd'} <= names
    assert 'AC_4' not in names and 'PW_3_4' not in names


# ---------------------------------------------------------------------------- arch.cuh on the host
def test_recurrence_equals_the_reference_arithmetic(harness):
    """The header's step, fed the normals the reference's arch() draws, gives its series bit for
    bit, NaN and inf included."""
    from elfi_b200.examples import arch
    rs = np.random.RandomState(7)
    B, n = 400, 100
    P = np.column_stack([rs.uniform(-1, 1, B), rs.uniform(0, 1, B)])
    P[:8] = [(0.3, 0.7), (1, 0), (1, 1), (-1, 0), (-1, 1), (0, 0), (-0.0, 0.5), (1.5, 3.0)]
    P[8:14] = [(np.nan, 0.5), (0.5, np.nan), (np.inf, 0.5), (0.5, np.inf), (0.5, -5.0),
               (-np.inf, -np.inf)]
    P[14:16] = [(1e300, 1.0), (1.0, 1e300)]
    xi = rs.randn(B, n + 1)
    e0 = rs.randn(B)
    xi[16, 5] = np.inf
    xi[17, 9] = np.nan
    e0[18] = -np.inf
    xi[19, 3:] = 0.0
    xi[20, 1] = -0.0
    with np.errstate(all='ignore'):
        want = arch.arch(P[:, 0], P[:, 1], n_obs=n, batch_size=B,
                         random_state=_GivenNormals(xi.copy(), e0.copy()))
    z = np.column_stack([e0, xi[:, 1:]])
    got = _rows(harness, P, z)
    assert _same_bits(got, want)
    assert np.isnan(got).any() and np.isinf(got).any()


def test_summaries_equal_numpy_at_every_n_and_lag(harness):
    rs = np.random.RandomState(3)
    for n in range(2, 129):
        x = rs.randn(12, n) * rs.uniform(1e-3, 1e3, (12, 1)) + rs.uniform(-50, 50, (12, 1))
        x[0] = 1.25                                   # constant
        x[1] = rs.choice([-0.0, 0.0], n)              # signed zeros
        x[2, rs.randint(n)] = np.nan
        x[3, rs.randint(n)] = np.inf
        x[4, rs.randint(n)] = -np.inf
        x[5] = np.round(x[5])                         # exact cancellations
        for L in range(1, min(8, n - 1) + 1):
            got = _summaries(harness, x, L)
            want = _reference_summaries(x, L)
            assert _same_bits(got, want), (n, L)


def test_summaries_equal_golden_crafted_rows(harness):
    g = load_golden('arch_summaries')
    for name, lags in (('crafted', (5, 8)), ('n2', (1,)), ('n128', (1, 8))):
        for L in lags:
            assert _same_bits(_summaries(harness, g[name], L), g['{}_L{}'.format(name, L)]), (name, L)


# ---------------------------------------------------------------------------- Python layer
@pytest.fixture
def arch_double(cpu_double, monkeypatch):
    import abi_double
    import arch_double
    import priors_double
    abi_double.install(monkeypatch, priors_double.TABLE, arch_double.TABLE)
    return cpu_double


def test_ops_validate_before_the_call(arch_double):
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    with pytest.raises(ValueError, match='n_obs'):
        ops.sim_arch(np.ones((2, 2)), n_obs=1)
    with pytest.raises(ValueError, match='n_obs'):
        ops.sim_arch(np.ones((2, 2)), n_obs=129)
    with pytest.raises(ValueError, match='n_lags'):
        ops.sim_arch(np.ones((2, 2)), n_lags=0)
    with pytest.raises(ValueError, match='n_lags'):
        ops.sim_arch(np.ones((2, 2)), n_lags=9)
    with pytest.raises(ValueError, match='n_lags'):
        ops.sim_arch(np.ones((2, 2)), n_obs=4, n_lags=4)
    with pytest.raises(ValueError, match='2 parameters'):
        ops.sim_arch(np.ones((2, 3)))
    with pytest.raises(ValueError, match='2 parameters'):
        ops.sim_arch(np.ones(2))
    with pytest.raises(ValueError, match='n_obs'):
        ops.arch_summaries(dev.to_device(np.ones((2, 129))))
    with pytest.raises(ValueError, match='n_lags'):
        ops.arch_summaries(dev.to_device(np.ones((2, 3))), n_lags=3)
    with pytest.raises(ValueError, match='batch, n'):
        ops.arch_summaries(dev.to_device(np.ones((2, 3, 4))))
    assert not arch_double.CALLS


def test_dispatch_host_device_and_lazy_agree(arch_double):
    """The four summary functions on host arrays, device tensors (a strided view included) and lazy
    simulator output give the same values; lags above the lazy output's are taken from its data."""
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    from elfi_b200.examples import arch
    rs = np.random.RandomState(0)
    full = rs.randn(6, 41)
    full[0] = 3.0
    y = full[:, 1:]
    fns = [arch.sample_mean, arch.sample_variance] + \
        [lambda x, i=i: arch.autocorr(x, i) for i in (1, 3, 6)] + \
        [lambda x, i=i, j=j: arch.pairwise_autocorr(x, i, j) for i, j in ((1, 2), (2, 5), (3, 3))]
    with np.errstate(all='ignore'):
        host = [f(y) for f in fns]
    for src in (dev.to_device(y), dev.to_device(full)[:, 1:]):
        for h, f in zip(host, fns):
            assert _same_bits(f(src).cpu().numpy(), h)
    S = ops.arch_summaries(y, n_lags=5).cpu().numpy()
    assert _same_bits(S, _reference_summaries(y, 5))
    lazy = arch.arch_device(0.3, 0.7, n_lags=2, batch_size=5, random_state=np.random.RandomState(1))
    data = lazy.materialize()
    assert tuple(data.shape) == (5, 100) and lazy.shape == (5, 100)
    with np.errstate(all='ignore'):
        for f in fns:
            assert _same_bits(f(lazy).cpu().numpy(), f(data.cpu().numpy()))
    Y, S2 = ops.sim_arch(np.tile([0.3, 0.7], (4, 1)), n_obs=30, n_lags=4, want_data=True)
    assert tuple(S2.shape) == (4, 12)
    assert _same_bits(S2.cpu().numpy(), _reference_summaries(Y.cpu().numpy(), 4))


def test_device_model_runs_rejection_and_smc(arch_double):
    import elfi_b200 as elfi
    from elfi_b200.examples import arch
    m, dp = arch.get_device_model(seed_obs=3, n_obs=60)
    assert dp.parameter_names == ['t1', 't2']
    assert dp.kinds == ['uniform', 'uniform']
    host = arch.get_model(seed_obs=3, n_obs=60)
    assert np.array_equal(m.observed['Y'], host.observed['Y'])
    res = elfi.Rejection(m['d'], batch_size=500, seed=1).sample(50, quantile=0.1, bar=False)
    assert res.n_samples == 50 and not np.any(np.isnan(res.discrepancies))
    smc = elfi.SMC(m['d'], batch_size=500, seed=2, device_proposal=dp).sample(
        50, quantiles=[0.5, 0.5], bar=False)
    assert len(smc.populations) == 2
    ss = [m[name] for name in ['MU', 'VAR', 'AC_1', 'AC_2', 'AC_3', 'AC_4', 'AC_5'] +
          ['PW_{}_{}'.format(i, j) for i, j in combinations(range(1, 6), 2)]]
    m['d'].become(elfi.AdaptiveDistance(*ss))
    ad = elfi.AdaptiveDistanceSMC(m['d'], batch_size=500, seed=3, device_proposal=dp).sample(
        50, rounds=2, quantile=0.5, bar=False)
    assert len(ad.populations) == 2
    assert 'elfi_b200_sim_arch_f64' in arch_double.CALLS
    with pytest.raises(ValueError, match='n_lags'):
        arch.get_device_model(n_lags=9)
