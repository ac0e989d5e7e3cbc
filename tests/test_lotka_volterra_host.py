"""CPU checks of the Lotka-Volterra example.

* the host path of elfi_b200.examples.lotka_volterra against the golden fixtures of the unmodified
  reference (tests/golden/gen_golden_lotka_volterra.py), bit for bit: draws (including return_full
  and the float64 switch after 20000 steps), summaries, Rejection;
* elfi_b200/csrc/lotka_volterra.cuh built for the host (tests/harness/lotka_volterra_harness.cpp):
  whole rows from given event draws against the host simulator fed the same draws (constructed
  sequences with event times exactly on grid times, extinctions, both species at 0, noise that
  truncates across 0, the cap), the int32 truncation, and the summaries against NumPy bit for bit
  for every n_obs in 3..128 and for constant rows;
* the Python layer (validation, dispatch, the throughput-mode graph and its prior) and the samplers
  on the CPU test double extended by tests/lv_double.py.
"""
import ctypes
import hashlib
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import load_golden

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope='module')
def harness(tmp_path_factory):
    gxx = shutil.which('g++')
    if gxx is None:
        pytest.skip('g++ not available')
    so = str(tmp_path_factory.mktemp('lv') / 'lotka_volterra_harness.so')
    subprocess.check_call([gxx, '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-o', so,
                           os.path.join(HERE, 'harness', 'lotka_volterra_harness.cpp')])
    lib = ctypes.CDLL(so)
    lib.harness_lv_row.restype = ctypes.c_int64
    return lib


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _summ(x, **kw):
    from elfi_b200.examples import lotka_volterra as lv
    with np.errstate(all='ignore'):
        return np.column_stack([
            lv.stock_mean(x, 0, **kw), lv.stock_mean(x, 1, **kw),
            lv.stock_log_variance(x, 0, **kw), lv.stock_log_variance(x, 1, **kw),
            lv.stock_autocorr(x, 0, 1, **kw), lv.stock_autocorr(x, 1, 1, **kw),
            lv.stock_autocorr(x, 0, 2, **kw), lv.stock_autocorr(x, 1, 2, **kw),
            lv.stock_crosscorr(x, **kw)])


def _sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), dtype=np.uint8)


# ---------------------------------------------------------------------------- reference goldens
def test_host_draws_match_reference_golden():
    from elfi_b200.examples import lotka_volterra as lv
    g = load_golden('lv_draws')
    x = lv.lotka_volterra(1.0, 0.005, 0.6, 50, 100, 0., n_obs=50, batch_size=3,
                          random_state=np.random.RandomState(1))
    assert x.dtype == np.int32 and np.array_equal(x, g['truth'])
    with np.errstate(all='ignore'):
        full = lv.lotka_volterra(*g['mixed_prm'].T, n_obs=30, batch_size=len(g['mixed_prm']),
                                 random_state=np.random.RandomState(2), return_full=True)
    assert np.array_equal(full[0], g['mixed'])
    for name, (stock, times) in (('mixed', full[2:]),):
        assert stock.shape == tuple(g[name + '_stock_shape'])
        assert str(stock.dtype) == str(g[name + '_stock_dtype'])
        assert np.array_equal(_sha(stock), g[name + '_stock_sha'])
        assert np.array_equal(_sha(times), g[name + '_times_sha'])
    # predators die out (rows 1, 2), start at 0 (row 3: the ramp), both species at 0 (row 4)
    assert np.all(g['mixed'][1:3, -1, 1] == 0) and np.all(g['mixed'][1:3, 0, 1] > 0)
    assert np.all(g['mixed'][3, :, 1] == 0) and g['mixed'][3, -1, 0] == 41
    assert np.all(g['mixed'][3, :-1, 0] == 40)
    assert np.all(g['mixed'][4] == 0)
    noisy = lv.lotka_volterra(*g['noisy_prm'].T, n_obs=25, batch_size=3,
                              random_state=np.random.RandomState(3))
    assert np.array_equal(noisy, g['noisy']) and (noisy < 0).any()
    so, to, stock, times = lv.lotka_volterra(1.0, 0.001, 1.0, 1000, 1000, n_obs=20, time_end=8.0,
                                             random_state=np.random.RandomState(4), return_full=True)
    assert np.array_equal(so, g['long']) and np.array_equal(to, g['long_times_out'])
    assert stock.shape == tuple(g['long_stock_shape']) and stock.shape[1] > 20001
    assert stock.dtype == np.float64 and str(g['long_stock_dtype']) == 'float64'
    assert np.array_equal(_sha(stock), g['long_stock_sha'])
    assert np.array_equal(_sha(times), g['long_times_sha'])
    assert np.array_equal(stock[:, -10:], g['long_stock_tail'])


def test_host_summaries_match_reference_golden():
    g = load_golden('lv_summaries')
    draws = load_golden('lv_draws')
    for name in ('truth', 'mixed', 'noisy', 'long'):
        assert np.array_equal(_summ(draws[name]), g[name], equal_nan=True), name
    for name in ('constant', 'n3', 'large', 'n128'):
        assert np.array_equal(_summ(g['x_' + name]), g[name], equal_nan=True), name
    assert np.isnan(g['constant'][0, 4:]).all() and np.isnan(g['constant'][1, [5, 7, 8]]).all()
    assert np.array_equal(_summ(draws['truth'], mu=3.5, std=0.25), g['truth_scaled'])


def test_rejection_matches_reference_golden(cpu_double):
    """Rejection on get_model (host simulator and summaries) reproduces the reference's sample."""
    import elfi_b200 as elfi
    from elfi_b200.examples import lotka_volterra as lv
    g = load_golden('lv_rejection')
    m = lv.get_model(seed_obs=7, time_end=0.5)
    assert np.array_equal(m.observed['LV'], g['observed'])
    res = elfi.Rejection(m['d'], batch_size=20, seed=3).sample(10, quantile=0.1, bar=False)
    assert res.n_sim == int(g['n_sim'])
    assert res.threshold == float(g['threshold'])
    assert np.array_equal(res.discrepancies, g['d'])
    for name in ('r1', 'r2', 'r3', 'prey0', 'predator0'):
        assert np.array_equal(res.samples[name], g['out_' + name]), name


def test_get_model_checks_true_params():
    from elfi_b200.examples import lotka_volterra as lv
    with pytest.raises(ValueError, match='six'):
        lv.get_model(true_params=[1.0, 0.005, 0.6, 50, 100], observation_noise=True)
    with pytest.raises(ValueError, match='five'):
        lv.get_model(true_params=[1.0, 0.005, 0.6, 50, 100, 1.0])
    m = lv.get_model(n_obs=10, observation_noise=True, seed_obs=1, time_end=1.0)
    assert sorted(m.parameter_names) == ['predator0', 'prey0', 'r1', 'r2', 'r3', 'sigma']


# ---------------------------------------------------------------------------- the header on the host
class _Draws:
    """A RandomState stand-in that hands the host simulator given draws: exponential(scale) is
    scale * E[k], uniform() is u[k], normal(scale) is scale * z (prey, then predators)."""

    def __init__(self, E, u, z):
        self.E, self.u, self.z = list(E), list(u), z
        self.k = 0
        self.j = 0

    def exponential(self, scale):
        e = self.E[self.k] if self.k < len(self.E) else 1.0
        return np.asarray(scale) * e

    def uniform(self, size):
        v = self.u[self.k] if self.k < len(self.u) else 0.5
        self.k += 1
        return np.full(size, v)

    def normal(self, scale, size):
        v = self.z[self.j]
        self.j += 1
        return np.asarray(scale) * v


def _row(harness, p, E, u, z, n_obs, time_end, max_events):
    t_out = np.linspace(0, time_end, n_obs)
    obs = np.empty((n_obs, 2))
    k = harness.harness_lv_row(_ptr(np.asarray(p, dtype=np.float64)), _ptr(E), _ptr(u), _ptr(z),
                               _ptr(t_out), ctypes.c_int32(n_obs), ctypes.c_double(time_end),
                               ctypes.c_int64(max_events), _ptr(obs))
    return obs, k


def _host_row(p, E, u, z, n_obs, time_end):
    from elfi_b200.examples import lotka_volterra as lv
    rs = _Draws(E, u, z[2:])
    with np.errstate(all='ignore'):
        so, _, _, times = lv.lotka_volterra(*p, n_obs=n_obs, time_end=time_end, random_state=rs,
                                            return_full=True)
    return so[0].astype(np.float64), int(np.argmax(times[0] >= time_end)), times[0]


def test_header_rows_match_host_simulator(harness):
    """Whole rows of the header (event, extinction time, emission, truncation) from given draws
    against the host simulator fed the same draws, bit for bit: random draws at several parameter
    points, and constructed rows whose event times fall exactly on grid times."""
    rs = np.random.RandomState(8)
    cases = []
    for p in ([1.0, 0.005, 0.6, 50, 100, 0.], [0.5, 0.05, 3.0, 10.0, 4.0, 0.],
              [1.0, 0.005, 0.6, 40.0, 0.5, 0.], [0.7, 0.005, 0.6, 0.3, 0.2, 0.],
              [1.0, 0.005, 0.6, 0.0, 30.0, 0.], [1.0, 0.005, 0.6, 3.0, 2.0, 10.0],
              [0.3, 0.01, 1.0, 1.0, 1.0, 25.0], [2.0, 0.01, 1.0, 20.7, 15.99, 0.5]):
        for _ in range(4):
            cases.append((p, rs.exponential(size=40000), rs.uniform(size=40000), 30.0, 16))
    # event times exactly on grid times: the reaction is always R1 (u = 0, r2 = 0), so the total
    # hazard of event k is r1 (X0 + k) + r3 Y = k + 2, and E_k = (k + 2) step / 2 makes most
    # waiting times exactly step / 2
    for n_obs in (5, 9, 17):
        time_end = 8.0
        step = time_end / (n_obs - 1)
        E = (np.arange(200) + 2.0) * (step / 2)
        for sigma in (0.0, 3.0):
            cases.append(([1.0, 0.0, 1.0, 1.0, 1.0, sigma], E, np.zeros(200), time_end, n_obs))
    n_ties = 0
    for p, E, u, time_end, n_obs in cases:
        z = rs.standard_normal(2 * n_obs)
        got, k = _row(harness, p, E, u, z, n_obs, time_end, E.size)
        want, kh, times = _host_row(p, E, u, z, n_obs, time_end)
        assert np.array_equal(got, want), (p, n_obs)
        assert k == kh, (p, k, kh)
        n_ties += np.isin(times[1:kh], np.linspace(0, time_end, n_obs)[1:-1]).sum()
    assert n_ties >= 12


def test_header_row_cap_and_invalid(harness):
    E, u, z = np.full(50, 0.01), np.full(50, 0.5), np.zeros(32)
    got, k = _row(harness, [1.0, 0.005, 0.6, 50, 100, 0.], E, u, z, 16, 30.0, 50)
    assert k == 50 and np.isnan(got).all()
    for p in ([-1.0, 0.005, 0.6, 50, 100, 0.], [1.0, np.nan, 0.6, 50, 100, 0.],
              [1.0, 0.005, 0.6, -0.5, 100, 0.], [1.0, 0.005, 0.6, 50, 2.0 ** 31, 0.],
              [1.0, 0.005, 0.6, 50, 100, -1.0]):
        got, k = _row(harness, p, E, u, z, 16, 30.0, 50)
        assert k == 0 and np.isnan(got).all(), p


def test_header_int32_truncation(harness):
    import lv_replay
    v = np.array([0.0, -0.0, 0.5, -0.5, 1.999, -1.999, 2147483647.9, 2147483648.0, -2147483648.9,
                  -2147483649.0, np.nan, np.inf, -np.inf, 1e300, -7.25, 3e9])
    out = np.empty_like(v)
    harness.harness_lv_to_int32(_ptr(v), ctypes.c_int64(v.size), _ptr(out))
    with np.errstate(invalid='ignore'):
        want = np.empty(v.size, dtype=np.int32)
        want[:] = v          # NumPy's float64 -> int32 assignment
    assert np.array_equal(out, want.astype(np.float64))
    assert np.array_equal(lv_replay.to_int32(v), out)


def test_header_summaries_match_numpy_every_n(harness):
    rs = np.random.RandomState(9)
    for n in range(3, 129):
        x = rs.randint(-50, 3000, (6, n, 2)).astype(np.float64)
        x[1] = 7.0                                  # constant rows
        x[2, :, 1] = 0.0
        x[3] = np.round(x[3] / 1000)                # ties
        x[4, :, 0] = rs.randint(-2 ** 31, 2 ** 31 - 1, n)
        S = np.empty((6, 9))
        harness.harness_lv_summaries(_ptr(x), ctypes.c_int64(6), ctypes.c_int32(n), _ptr(S))
        assert np.array_equal(S, _summ(x), equal_nan=True), n
        assert np.array_equal(_summ(x), _summ(x.astype(np.int32)), equal_nan=True), n


# ---------------------------------------------------------------------------- Python layer
@pytest.fixture
def lv_double(cpu_double, monkeypatch):
    import abi_double
    import lv_double
    import priors_double
    abi_double.install(monkeypatch, priors_double.TABLE, lv_double.TABLE)
    return cpu_double


def test_ops_validate_before_the_call(lv_double):
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    P = np.tile([1.0, 0.005, 0.6, 50, 100, 0.], (3, 1))
    with pytest.raises(ValueError, match='1 <= n_obs <= 1024'):
        ops.sim_lotka_volterra(P, n_obs=1025)
    with pytest.raises(ValueError, match='time_end'):
        ops.sim_lotka_volterra(P, time_end=0.0)
    with pytest.raises(ValueError, match='time_end'):
        ops.sim_lotka_volterra(P, time_end=np.inf)
    with pytest.raises(ValueError, match='max_events'):
        ops.sim_lotka_volterra(P, max_events=2 ** 32)
    with pytest.raises(ValueError, match='max_events'):
        ops.sim_lotka_volterra(P, max_events=0)
    with pytest.raises(ValueError, match='parameter width of 5'):
        ops.sim_lotka_volterra(P[:, :5])
    with pytest.raises(ValueError, match='3 <= n_obs <= 128'):
        ops.lv_summaries(dev.to_device(np.zeros((2, 129, 2))))
    with pytest.raises(ValueError, match='3 <= n_obs <= 128'):
        ops.lv_summaries(dev.to_device(np.zeros((2, 2, 2))))
    with pytest.raises(ValueError, match='batch, n_obs, 2'):
        ops.lv_summaries(dev.to_device(np.zeros((2, 10, 3))))
    assert not lv_double.CALLS
    obs, n = ops.sim_lotka_volterra(P, n_obs=1024, time_end=1.0)
    assert tuple(obs.shape) == (3, 1024, 2) and tuple(n.shape) == (3,)


def test_dispatch_host_device_and_lazy_agree(lv_double):
    """The summaries on host arrays, device tensors and lazy simulator output agree."""
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    from elfi_b200.examples import lotka_volterra as lv
    x = load_golden('lv_draws')['truth']
    h = _summ(x)
    assert np.array_equal(ops.lv_summaries(x).cpu().numpy(), h)
    fns = [lambda s: lv.stock_mean(s, 0), lambda s: lv.stock_mean(s, 1),
           lambda s: lv.stock_log_variance(s, 0), lambda s: lv.stock_log_variance(s, 1),
           lambda s: lv.stock_autocorr(s, 0, 1), lambda s: lv.stock_autocorr(s, 1, 1),
           lambda s: lv.stock_autocorr(s, 0, 2), lambda s: lv.stock_autocorr(s, 1, 2),
           lv.stock_crosscorr]
    xd = dev.to_device(x.astype(np.float64))
    for c, fn in enumerate(fns):
        assert np.array_equal(fn(xd).cpu().numpy(), h[:, c]), c
    assert np.array_equal(lv.stock_mean(xd, 1, mu=2.0, std=4.0).cpu().numpy(),
                          lv.stock_mean(x, 1, mu=2.0, std=4.0))
    with pytest.raises(ValueError, match='lags'):
        lv.stock_autocorr(xd, 0, lag=3)
    lazy = lv.lotka_volterra_device(1.0, 0.005, 0.6, 50, 100, n_obs=20, time_end=5.0,
                                    batch_size=4, random_state=np.random.RandomState(1))
    assert lazy.shape == (4, 20, 2)
    data = lazy.materialize()
    assert data is lazy.materialize()
    hd = data.cpu().numpy()
    assert np.all(hd[:, 0] == [50, 100])
    for c, fn in enumerate(fns):
        assert np.array_equal(fn(lazy).cpu().numpy(), _summ(hd)[:, c]), c
    assert lv_double.CALLS.count('elfi_b200_sim_lotka_volterra_f64') == 1
    with pytest.raises(ValueError, match='full event history'):
        lv.lotka_volterra_device(1.0, 0.005, 0.6, return_full=True)
    obs, n = ops.sim_lotka_volterra(np.array([[-1.0, 0.005, 0.6, 50, 100, 0.],
                                              [1.0, 0.005, 0.6, 50, 100, 0.]]), time_end=5.0)
    obs, n = obs.cpu().numpy(), n.cpu().numpy()
    assert np.isnan(obs[0]).all() and n[0] == 0 and np.isfinite(obs[1]).all() and n[1] > 0


def test_device_prior_matches_host_prior(lv_double):
    """DeviceProposal: the sorted parameter names, the box where the prior density is positive,
    and logpdf == the host ModelPrior's, including -inf outside the box and at x <= 0."""
    from elfi_b200.examples import lotka_volterra as lv
    from elfi_b200.samplers import ModelPrior
    for noise in (False, True):
        host = ModelPrior(lv.get_model(n_obs=10, observation_noise=noise, seed_obs=1, time_end=1.0))
        m, dp = lv.get_device_model(n_obs=10, observation_noise=noise, seed_obs=1, time_end=1.0)
        assert dp.parameter_names == list(host.parameter_names)
        p = len(dp.parameter_names)
        rs = np.random.RandomState(2)
        x = np.empty((400, p))
        for i, name in enumerate(dp.parameter_names):
            lo, hi = dp.box[0][i], dp.box[1][i]
            if np.isfinite(lo):
                x[:, i] = np.exp(rs.uniform(np.log(lo) - 0.5, np.log(hi) + 0.5, 400))
                x[:5, i] = [lo, hi, 0.0, -1.0, np.nextafter(lo, 0)]
                assert np.isclose(lo, np.exp(-6.0) if name != 'sigma' else 0.5)
            else:
                x[:, i] = rs.normal(80, 30, 400)
        got = dp.logpdf(x).cpu().numpy()
        want = host.logpdf(x)
        assert np.array_equal(np.isinf(got), np.isinf(want))
        fin = np.isfinite(want)
        assert fin.sum() > 50 and (~fin).sum() > 50
        assert np.allclose(got[fin], want[fin], rtol=1e-13, atol=1e-13)
        draws = dp.rvs(x[fin][:20], np.eye(p) * 0.01, None, 200, key=3).cpu().numpy()
        assert np.isfinite(host.logpdf(draws)).all()


def test_device_model_runs_rejection_and_smc(lv_double):
    import elfi_b200 as elfi
    from elfi_b200.examples import lotka_volterra as lv
    m, dp = lv.get_device_model(seed_obs=3, time_end=0.5, max_events=5000)
    host_m = lv.get_model(seed_obs=3, time_end=0.5)
    assert np.array_equal(m.observed['LV'], host_m.observed['LV'])
    assert dp.parameter_names == ['predator0', 'prey0', 'r1', 'r2', 'r3']
    assert sorted(n for n in m.nodes if not n.startswith('_')) == sorted(
        n for n in host_m.nodes if not n.startswith('_'))
    with pytest.raises(ValueError, match='3 <= n_obs <= 128'):
        lv.get_device_model(n_obs=200)
    res = elfi.Rejection(m['d'], batch_size=50, seed=1).sample(5, quantile=0.1, bar=False)
    assert res.n_samples == 5 and not np.any(np.isnan(res.discrepancies))
    smc = elfi.SMC(m['d'], batch_size=50, seed=2, device_proposal=dp).sample(
        5, quantiles=[0.5, 0.5], bar=False)
    assert len(smc.populations) == 2
    assert 'elfi_b200_sim_lotka_volterra_f64' in lv_double.CALLS
    assert 'elfi_b200_lv_summaries_f64' in lv_double.CALLS
