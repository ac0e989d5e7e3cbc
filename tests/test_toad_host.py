"""CPU checks of the toad example.

* the host path of elfi_b200.examples.toad against the golden fixtures of the unmodified reference
  (tests/golden/gen_golden_toad.py), bit for bit: draws, summaries, Rejection;
* elfi_b200/csrc/toad.cuh built for the host (tests/harness/toad_harness.cpp): the quantile picks and
  both median paths for every kept count 1 .. 4096 against NumPy, the exp(-20) floor, the
  nan_to_num mapping, the refuge day and the levy_stable step including its alpha == 1 branch;
* the Python layer (validation, dispatch, the throughput-mode graph) and the samplers on the CPU
  test double extended by tests/toad_double.py.
"""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import load_golden

HERE = os.path.dirname(os.path.abspath(__file__))
P11 = np.linspace(0, 1, 11)


@pytest.fixture(scope='module')
def harness(tmp_path_factory):
    gxx = shutil.which('g++')
    if gxx is None:
        pytest.skip('g++ not available')
    so = str(tmp_path_factory.mktemp('toad') / 'toad_harness.so')
    subprocess.check_call([gxx, '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-o', so,
                           os.path.join(HERE, 'harness', 'toad_harness.cpp')])
    lib = ctypes.CDLL(so)
    lib.harness_toad_floor.restype = ctypes.c_double
    return lib


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _summ(x, lag, p=P11, thd=10):
    from elfi_b200.examples import toad
    with np.errstate(all='ignore'):
        return toad.compute_summaries(x, lag, p=p, thd=thd)


# ---------------------------------------------------------------------------- reference goldens
def test_host_draws_match_reference_golden():
    from elfi_b200.examples import toad
    g = load_golden('toad_draws')
    prm = g['prm']
    x = toad.toad(*prm.T, n_toads=5, n_days=9, batch_size=len(prm),
                  random_state=np.random.RandomState(3))
    assert np.array_equal(x, g['x'], equal_nan=True)
    # alpha == 1 with gamma == 0 in a mixed batch: NaN steps; elsewhere finite
    assert np.isnan(x[1:, :, 0]).all() and np.isfinite(x[:, :, 2:]).all()
    with np.errstate(all='ignore'):
        xz = toad.toad(*g['zero_gamma_prm'].T, n_toads=5, n_days=9, batch_size=2,
                       random_state=np.random.RandomState(4))
    assert np.array_equal(xz, g['x_zero_gamma'], equal_nan=True)
    xt = toad.toad(1.7, 35.0, 0.6, batch_size=3, random_state=np.random.RandomState(5))
    assert np.array_equal(xt, g['x_true']) and xt.shape == (63, 66, 3)


def test_host_raises_where_the_reference_raises():
    from elfi_b200.examples import toad
    for prm in ((2.5, 10.0, 0.5), (0.0, 10.0, 0.5), (1.5, -1.0, 0.5)):
        with pytest.raises(ValueError):
            toad.toad(*prm, n_toads=3, n_days=3, random_state=np.random.RandomState(0))


def test_host_summaries_match_reference_golden():
    g = load_golden('toad_summaries')
    draws = load_golden('toad_draws')
    for lag in range(1, 9):
        assert np.array_equal(_summ(draws['x'], lag), g['draws_lag{}'.format(lag)]), lag
    for lag in (1, 2, 4, 8):
        assert np.array_equal(_summ(draws['x_true'], lag), g['true_lag{}'.format(lag)]), lag
    names = [k[2:] for k in g if k.startswith('x_')]
    assert len(names) == 10
    for n in names:
        got = _summ(g['x_' + n], int(g['lag_' + n]), g['p_' + n], float(g['thd_' + n]))
        assert np.array_equal(got, g['s_' + n]), n
    assert np.all(g['s_returned'][:, 0] == 40) and np.all(g['s_returned'][:, 1:] == np.inf)
    # 11 kept values of 1.5e308: the masked median doubles it (inf -> DBL_MAX), np.median does not
    assert g['s_big54'][0, 1] == np.finfo(float).max and g['s_big55'][0, 1] == 1.5e308


def test_rejection_matches_reference_golden(cpu_double):
    """Rejection on get_model (host simulator and summaries) reproduces the reference's sample."""
    import elfi_b200 as elfi
    from elfi_b200.examples import toad
    g = load_golden('toad_rejection')
    m = toad.get_model(seed_obs=7)
    assert np.array_equal(m.observed['toad'], g['observed'])
    res = elfi.Rejection(m['d'], batch_size=10, seed=3).sample(10, bar=False)
    assert res.n_sim == int(g['n_sim'])
    assert res.threshold == float(g['threshold'])
    assert np.array_equal(res.discrepancies, g['d'])
    for name in ('alpha', 'gamma', 'p0'):
        assert np.array_equal(res.samples[name], g['out_' + name]), name


# ---------------------------------------------------------------------------- toad.cuh on the host
def test_header_quantiles_and_medians_every_count(harness):
    """For every kept count n = 1 .. 4096: the p quantiles equal np.nanquantile and the median
    equals np.nanmedian of a column of n kept values among n_rows rows, below (masked median) and
    from 600 rows (np.median); values with ties, infinities and 1.5e308."""
    rs = np.random.RandomState(1)
    levels = [P11, np.array([0.0, 0.05, 1 / 3, 0.5, 0.999, 1.0])]
    for n in range(1, 4097):
        v = np.sort(np.round(rs.standard_cauchy(n) * 50, 1 if n % 3 else 3) ** 2)
        if n % 7 == 0:
            v[-1] = np.inf
        if n % 11 == 0:
            v[:] = 1.5e308
        p = levels[n % 2]
        out = np.empty(p.size + 1)
        for n_rows in {max(n, 599), max(n, 600)} if n < 600 else {n}:
            harness.harness_toad_quantiles(_ptr(v), ctypes.c_int32(n), ctypes.c_int32(n_rows),
                                           ctypes.c_int32(p.size), _ptr(p), _ptr(out))
            col = np.full((n_rows, 1), np.nan)
            col[rs.permutation(n_rows)[:n], 0] = rs.permutation(v)
            with np.errstate(all='ignore'):
                want_q = np.nanquantile(col, p, axis=0)[:, 0]
                want_m = np.nanmedian(col, axis=0)[0]
            assert np.array_equal(out[:-1], want_q, equal_nan=True), (n, n_rows)
            assert np.array_equal(out[-1:], [want_m], equal_nan=True), (n, n_rows)


def test_header_floor_log_and_nan_to_num(harness):
    assert harness.harness_toad_floor() == np.exp(-20)
    f = np.exp(-20)
    lo = np.array([0.0, 1.0, 1.0, 5.0, np.inf, 1.0, np.nan, 0.0, -np.inf, 3.0])
    hi = np.array([0.0, 1.0 + f / 2, 1.0 + 2 * f, 7.5, np.inf, np.inf, 1.0, 1e308, 1.0, 2.0])
    x = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, 1.5e308, -3.0, 5e-324, 1.0, np.nan])
    out, raw = np.empty(lo.size), np.empty(lo.size)
    harness.harness_toad_post(_ptr(lo), _ptr(hi), _ptr(x), ctypes.c_int64(lo.size), _ptr(out),
                              _ptr(raw))
    with np.errstate(all='ignore'):
        want = np.nan_to_num(np.log(np.maximum(hi - lo, np.exp(-20))), nan=np.inf)
    assert np.allclose(out, want, rtol=4e-16, atol=0) or np.array_equal(out, want)
    assert np.array_equal(out[[0, 1, 4, 5, 6, 8, 9]], want[[0, 1, 4, 5, 6, 8, 9]])
    assert np.array_equal(raw, np.nan_to_num(x, nan=np.inf))
    assert raw[1] == np.finfo(float).max and raw[2] == -np.finfo(float).max


def test_header_refuge_day(harness):
    import toad_replay as tr
    rs = np.random.RandomState(3)
    w = rs.randint(0, 2 ** 63, 5000, dtype=np.uint64) * np.uint64(2) + rs.randint(0, 2, 5000).astype(np.uint64)
    w[:3] = [0, 2 ** 64 - 1, 2 ** 63]
    d = rs.randint(1, 2 ** 31 - 1, 5000).astype(np.int32)
    d[:3] = [1, 2 ** 31 - 1, 62]
    out = np.empty(5000, dtype=np.int32)
    harness.harness_toad_refuge(_ptr(w), _ptr(d), ctypes.c_int64(5000), _ptr(out))
    want = np.array([(int(a) * int(b)) >> 64 for a, b in zip(w, d)])
    assert np.array_equal(out, want) and np.array_equal(tr.refuge_day(w, d), want)
    assert np.all((out >= 0) & (out < d))


def test_header_step_matches_scipy_formula(harness):
    """The step of toad.cuh against the replay's NumPy restatement of SciPy (glibc and NumPy may
    differ by an ulp in sin / cos / tan / pow / log) and the alpha == 1 branch (NaN at
    gamma == 0); gamma == 0 gives zero steps otherwise."""
    import toad_replay as tr
    rs = np.random.RandomState(4)
    n = 20000
    alpha = rs.uniform(1, 2, n)
    alpha[:2000] = 1.0
    alpha[2000:2100] = 2.0
    gamma = rs.uniform(0, 100, n)
    gamma[::97] = 0.0
    u, v = rs.uniform(0, 1, n), 1.0 - rs.uniform(0, 1, n)
    out = np.empty(n)
    harness.harness_toad_step(_ptr(alpha), _ptr(gamma), _ptr(u), _ptr(v), ctypes.c_int64(n),
                              _ptr(out))
    want, c1, c2 = tr.step(alpha, gamma, u, v)
    one = alpha == 1
    assert np.isnan(out[one & (gamma == 0)]).all()
    assert np.array_equal(np.isnan(out), np.isnan(want))
    ok = np.abs(out - want) <= tr.step_bound(want, alpha, c1, c2)
    assert ok[~np.isnan(want)].all(), np.argwhere(~ok)[:5]
    assert np.all(out[~one & (gamma == 0)] == 0)


# ---------------------------------------------------------------------------- Python layer
@pytest.fixture
def toad_double(cpu_double, monkeypatch):
    import abi_double
    import priors_double
    import toad_double
    abi_double.install(monkeypatch, priors_double.TABLE, toad_double.TABLE)
    return cpu_double


def test_ops_validate_before_the_call(toad_double):
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    P = np.tile([1.7, 35.0, 0.6], (3, 1))
    x = dev.to_device(np.zeros((63, 66, 2)))
    with pytest.raises(ValueError, match='n_toads \\* \\(n_days - lag\\)'):
        ops.sim_toad(P, n_toads=67)
    with pytest.raises(ValueError, match='lag'):
        ops.sim_toad(P, lags=(1, 63))
    with pytest.raises(ValueError, match='at most 8 lags'):
        ops.sim_toad(P, lags=tuple(range(1, 10)))
    with pytest.raises(ValueError, match='quantile levels'):
        ops.sim_toad(P, p=np.linspace(0, 1, 33))
    with pytest.raises(ValueError, match='in \\[0, 1\\]'):
        ops.toad_summaries(x, 1, p=[0.5, 1.5])
    with pytest.raises(ValueError, match='n_days \\* n_toads'):
        ops.sim_toad(P, n_toads=2 ** 16, n_days=2 ** 15 + 1, lags=None)
    with pytest.raises(ValueError, match='parameter width of 2'):
        ops.sim_toad(np.ones((3, 2)))
    with pytest.raises(ValueError, match='lag'):
        ops.toad_summaries(x, 0)
    with pytest.raises(ValueError, match='n_toads \\* \\(n_days - lag\\)'):
        ops.toad_summaries(dev.to_device(np.zeros((100, 66, 2))), 1)
    with pytest.raises(ValueError, match='n_days, n_toads, batch'):
        ops.toad_summaries(dev.to_device(np.zeros((63, 66))), 1)
    assert not toad_double.CALLS
    # the data alone may go beyond the summaries' limit
    X, S = ops.sim_toad(P[:1], n_toads=100, n_days=100, want_data=True, lags=None)
    assert tuple(X.shape) == (1, 100, 100) and S is None


def test_dispatch_host_device_and_lazy_agree(toad_double):
    """compute_summaries on host arrays, device tensors and lazy simulator output agree."""
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    from elfi_b200.examples import toad
    x = load_golden('toad_draws')['x_true']
    for lag in (1, 2, 4, 8, 3):
        h = _summ(x, lag)
        assert np.array_equal(toad.compute_summaries(dev.to_device(x), lag).cpu().numpy(), h)
    assert np.array_equal(ops.toad_summaries(x, 2, p=[0.2, 0.7], thd=3.0).cpu().numpy(),
                          _summ(x, 2, p=np.array([0.2, 0.7]), thd=3.0))
    lazy = toad.toad_device(1.7, 35.0, 0.6, batch_size=4, random_state=np.random.RandomState(1))
    data = lazy.materialize()
    assert tuple(data.shape) == (63, 66, 4) and lazy.shape == (63, 66, 4)
    hd = data.cpu().numpy()
    assert np.all(hd[0] == 0)
    for lag in (1, 2, 4, 8, 5):
        assert np.array_equal(toad.compute_summaries(lazy, lag).cpu().numpy(), _summ(hd, lag)), lag
    assert np.array_equal(toad.compute_summaries(lazy, 2, thd=4).cpu().numpy(), _summ(hd, 2, thd=4))
    X, S = ops.sim_toad(np.array([[2.5, 1.0, 0.5], [1.5, -1.0, 0.5], [1.5, 1.0, 0.5]]), want_data=True)
    X = X.cpu().numpy()
    assert np.isnan(X[:2]).all() and np.isfinite(X[2]).all()
    assert np.all(S.cpu().numpy()[:2, 0::12] == 0)


def test_device_model_runs_rejection_and_smc(toad_double):
    import elfi_b200 as elfi
    from elfi_b200.examples import toad
    m, dp = toad.get_device_model(seed_obs=3)
    host_m = toad.get_model(seed_obs=3)
    assert np.array_equal(m.observed['toad'], host_m.observed['toad'])
    assert dp.parameter_names == ['alpha', 'gamma', 'p0']
    assert dp.kinds == ['uniform', 'uniform', 'uniform']
    assert sorted(n for n in m.nodes if not n.startswith('_')) == sorted(
        n for n in host_m.nodes if not n.startswith('_'))
    res = elfi.Rejection(m['d'], batch_size=50, seed=1).sample(5, quantile=0.1, bar=False)
    assert res.n_samples == 5 and not np.any(np.isnan(res.discrepancies))
    smc = elfi.SMC(m['d'], batch_size=50, seed=2, device_proposal=dp).sample(
        5, quantiles=[0.5, 0.5], bar=False)
    assert len(smc.populations) == 2
    assert 'elfi_b200_sim_toad_f64' in toad_double.CALLS
