"""CPU checks of the Lorenz example.

* the host path of elfi_b200.examples.lorenz against the golden fixtures of the unmodified reference
  (tests/golden/gen_golden_lorenz.py), bit for bit: draws, noise-free trajectories, summaries,
  Rejection; and the reference's raises;
* elfi_b200/csrc/lorenz.cuh built for the host (tests/harness/lorenz_harness.cpp): whole phi = 1
  trajectories, single steps with a given eta, and the six summaries bit for bit against NumPy;
* the Python layer (validation, dispatch, the throughput-mode graph) and the samplers on the CPU
  test double extended by tests/lorenz_double.py.
"""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import load_golden

HERE = os.path.dirname(os.path.abspath(__file__))
SUMMARY_T = list(range(2, 21)) + [159, 160, 161]
SUMMARY_M = [2, 3, 4, 5, 7, 8, 9, 17, 40, 64, 128]


@pytest.fixture(scope='module')
def harness(tmp_path_factory):
    gxx = shutil.which('g++')
    if gxx is None:
        pytest.skip('g++ not available')
    so = str(tmp_path_factory.mktemp('lorenz') / 'lorenz_harness.so')
    subprocess.check_call([gxx, '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-o', so,
                           os.path.join(HERE, 'harness', 'lorenz_harness.cpp')])
    return ctypes.CDLL(so)


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _run(harness, init, T, th1, th2, f=10.0, dt=4 / 160, eta=None):
    init = np.ascontiguousarray(init, dtype=np.float64)
    m = init.size
    out = np.empty((T, m))
    if eta is not None:
        eta = np.ascontiguousarray(eta, dtype=np.float64)
    harness.harness_lorenz_run(_ptr(init), ctypes.c_int32(m), ctypes.c_int32(T), ctypes.c_double(th1),
                               ctypes.c_double(th2), ctypes.c_double(f), ctypes.c_double(dt),
                               None if eta is None else _ptr(eta), _ptr(out))
    return out


def _summ_harness(harness, x):
    B, T, m = x.shape
    out = np.empty((B, 6))
    s = [v // 8 for v in x.strides]
    harness.harness_lorenz_summaries(_ptr(x), ctypes.c_int64(s[0]), ctypes.c_int64(s[1]),
                                     ctypes.c_int64(s[2]), ctypes.c_int64(B), ctypes.c_int32(T),
                                     ctypes.c_int32(m), _ptr(out))
    return out


def _summ_numpy(x):
    from elfi_b200.examples import lorenz
    with np.errstate(all='ignore'):
        return np.column_stack([lorenz.mean(x), lorenz.var(x), lorenz.autocov(x), lorenz.cov(x),
                                lorenz.xcov(x, True), lorenz.xcov(x, False)])


# ---------------------------------------------------------------------------- reference goldens
def test_host_draws_match_reference_golden():
    from elfi_b200.examples import lorenz
    g = load_golden('lorenz_draws')
    prm = g['prm']
    x = lorenz.forecast_lorenz(*prm.T, n_timestep=16, total_duration=0.4, batch_size=len(prm),
                               random_state=np.random.RandomState(3))
    assert np.array_equal(x, g['x']) and np.isfinite(x).all()
    assert np.array_equal(g['x'][:, 0], np.tile(lorenz.INITIAL_STATE, (len(prm), 1)))
    with np.errstate(invalid='ignore'):
        xnan = lorenz.forecast_lorenz(2.0, 0.1, phi=1.5, n_timestep=4, batch_size=2,
                                      random_state=np.random.RandomState(4))
    assert np.array_equal(xnan, g['x_phi15'], equal_nan=True) and np.isnan(xnan[:, 1:]).all()
    fp = g['noise_free_prm']
    xf = lorenz.forecast_lorenz(*fp.T, phi=1.0, batch_size=len(fp),
                                random_state=np.random.RandomState(5))
    assert np.array_equal(xf, g['x_noise_free'])


def test_host_raises_where_the_reference_raises():
    from elfi_b200.examples import lorenz
    with pytest.raises(ValueError):
        lorenz.forecast_lorenz(2.0, 0.1, n_obs=41, n_timestep=3)
    with pytest.raises(ValueError):
        lorenz.forecast_lorenz(2.0, 0.1, n_timestep=3, initial_state=np.array(lorenz.INITIAL_STATE))
    with pytest.raises(AttributeError):
        lorenz.forecast_lorenz(2.0, 0.1, n_timestep=3, initial_state=list(lorenz.INITIAL_STATE))


def test_host_summaries_match_reference_golden():
    g = load_golden('lorenz_summaries')
    draws = load_golden('lorenz_draws')
    assert np.array_equal(_summ_numpy(draws['x']), g['draws'])
    assert np.array_equal(_summ_numpy(draws['x_noise_free']), g['noise_free'])
    crafted = [k[2:] for k in g if k.startswith('x_')]
    assert len(crafted) == 6
    for name in crafted:
        assert np.array_equal(_summ_numpy(g['x_' + name]), g['s_' + name], equal_nan=True), name
    s40 = g['s_m40']      # row 0 holds a NaN, row 1 a +inf, row 3 is constant
    assert np.isnan(s40[0]).all() and not np.isfinite(s40[1]).any() and np.all(s40[3, 1:] == 0)


def test_rejection_matches_reference_golden(cpu_double):
    """Rejection on get_model (host simulator and summaries) reproduces the reference's sample."""
    import elfi_b200 as elfi
    from elfi_b200.examples import lorenz
    g = load_golden('lorenz_rejection')
    m = lorenz.get_model(seed_obs=7)
    assert np.array_equal(m.observed['Lorenz'], g['observed'])
    res = elfi.Rejection(m['d'], batch_size=10, seed=3).sample(10, bar=False)
    assert res.n_sim == int(g['n_sim'])
    assert res.threshold == float(g['threshold'])
    assert np.array_equal(res.discrepancies, g['d'])
    for name in ('theta1', 'theta2'):
        assert np.array_equal(res.samples[name], g['out_' + name]), name


# ---------------------------------------------------------------------------- lorenz.cuh on the host
def test_header_noise_free_trajectories_equal_reference(harness):
    """phi = 1 keeps eta at 0: all 160 steps of the header's RK4 equal the reference's bits."""
    from elfi_b200.examples import lorenz
    g = load_golden('lorenz_draws')
    for (th1, th2), want in zip(g['noise_free_prm'], g['x_noise_free']):
        assert np.array_equal(_run(harness, lorenz.INITIAL_STATE, 160, th1, th2), want)


@pytest.mark.parametrize('m', [4, 5, 40, 41, 65, 128])
def test_header_steps_equal_numpy(harness, m):
    """Single steps with a given eta, and whole eta = 0 runs, for ring sizes the reference's
    default state does not cover (NumPy restated with np.roll, see examples.lorenz._lorenz_ode)."""
    import lorenz_replay as lr
    rs = np.random.RandomState(m)
    init = rs.randn(m) * 4
    for th1, th2 in ((2.0, 0.1), (0.5, 0.0), (3.5, 0.3)):
        eta = rs.randn(1, m)
        got = _run(harness, init, 2, th1, th2, eta=eta)
        want = lr.rk4_step(init[None, :], eta, np.array([th1]), np.array([th2]), 10.0, 4 / 160)
        assert np.array_equal(got[1], want[0])
        run = _run(harness, init, 40, th1, th2)
        y = init[None, :]
        for s in range(1, 40):
            y = lr.rk4_step(y, np.zeros((1, m)), np.array([th1]), np.array([th2]), 10.0, 4 / 160)
            assert np.array_equal(run[s], y[0]), s


def test_header_ar1_equals_numpy(harness):
    rs = np.random.RandomState(2)
    eta, e = rs.randn(1000), rs.randn(1000)
    for phi in (0.0, 0.984, 1.0):
        s = float(np.sqrt(1 - pow(phi, 2)))
        out = np.empty(1000)
        harness.harness_lorenz_ar1(_ptr(eta), _ptr(e), ctypes.c_int64(1000), ctypes.c_double(phi),
                                   ctypes.c_double(s), _ptr(out))
        assert np.array_equal(out, phi * eta + e * s)


@pytest.mark.parametrize('m', SUMMARY_M)
def test_header_summaries_equal_numpy(harness, m):
    """Every T in 2..20, 159, 160, 161: the flattened runs (T - 1) m and T m cross NumPy's pairwise
    leaf boundaries; a strided view gives the bits of its contiguous copy."""
    rs = np.random.RandomState(m)
    for T in SUMMARY_T:
        x = rs.randn(3, T, m) * 10 ** rs.uniform(-3, 3, (3, T, m))
        assert np.array_equal(_summ_harness(harness, x), _summ_numpy(x)), T
    big = rs.randn(2, 161, m + 3)[:, ::-1, 1:m + 1]
    assert np.array_equal(_summ_harness(harness, big), _summ_numpy(np.ascontiguousarray(big)))


def test_header_summaries_nan_inf_constant(harness):
    g = load_golden('lorenz_summaries')
    for name in [k[2:] for k in g if k.startswith('x_')]:
        with np.errstate(all='ignore'):
            got = _summ_harness(harness, np.ascontiguousarray(g['x_' + name]))
        assert np.array_equal(got, g['s_' + name], equal_nan=True), name


# ---------------------------------------------------------------------------- Python layer
@pytest.fixture
def lorenz_double(cpu_double, monkeypatch):
    import abi_double
    import lorenz_double
    import priors_double
    abi_double.install(monkeypatch, priors_double.TABLE, lorenz_double.TABLE)
    return cpu_double


def test_ops_validate_before_the_call(lorenz_double):
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    P = np.tile([2.0, 0.1], (3, 1))
    with pytest.raises(ValueError, match='n_obs'):
        ops.sim_lorenz(P, initial_state=np.ones(3))
    with pytest.raises(ValueError, match='n_obs'):
        ops.sim_lorenz(P, initial_state=np.ones(129))
    with pytest.raises(ValueError, match='one vector'):
        ops.sim_lorenz(P, initial_state=np.ones((2, 40)))
    with pytest.raises(ValueError, match='n_timestep'):
        ops.sim_lorenz(P, n_timestep=1)
    with pytest.raises(ValueError, match='n_timestep \\* n_obs'):
        ops.sim_lorenz(P, n_timestep=241, initial_state=np.ones(128))
    with pytest.raises(ValueError, match='parameter width of 3'):
        ops.sim_lorenz(np.ones((3, 3)))
    with pytest.raises(ValueError, match='n_obs'):
        ops.lorenz_summaries(dev.to_device(np.ones((2, 5, 129))))
    with pytest.raises(ValueError, match='2 <= n_obs'):
        ops.lorenz_summaries(dev.to_device(np.ones((2, 5, 1))))
    with pytest.raises(ValueError, match='n_timestep'):
        ops.lorenz_summaries(dev.to_device(np.ones((2, 1, 40))))
    with pytest.raises(ValueError, match='batch, n_timestep, n_obs'):
        ops.lorenz_summaries(dev.to_device(np.ones((2, 40))))
    assert not lorenz_double.CALLS
    # the summaries alone may stop at the limit; the data can go beyond it
    X, S = ops.sim_lorenz(P[:1], n_timestep=241, initial_state=np.ones(128), want_data=True,
                          want_summaries=False)
    assert tuple(X.shape) == (1, 241, 128) and S is None


def test_dispatch_host_device_and_lazy_agree(lorenz_double):
    """The summaries on host arrays, device tensors and lazy simulator output give the same values."""
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    from elfi_b200.examples import lorenz
    fns = (lorenz.mean, lorenz.var, lorenz.autocov, lorenz.cov, lambda x: lorenz.xcov(x, True),
           lambda x: lorenz.xcov(x, False))
    x = load_golden('lorenz_draws')['x']
    host = [f(x) for f in fns]
    for h, f in zip(host, fns):
        assert np.array_equal(f(dev.to_device(x)).cpu().numpy(), h)
    assert np.array_equal(ops.lorenz_summaries(x).cpu().numpy(), np.column_stack(host))
    lazy = lorenz.lorenz_device(2.0, 0.1, n_timestep=20, batch_size=4,
                                random_state=np.random.RandomState(1))
    data = lazy.materialize()
    assert tuple(data.shape) == (4, 20, 40) and lazy.shape == (4, 20, 40)
    assert np.array_equal(data[:, 0].cpu().numpy(), np.tile(lorenz.INITIAL_STATE, (4, 1)))
    for f in fns:
        assert np.array_equal(f(lazy).cpu().numpy(), f(data.cpu().numpy()))
    X, S = ops.sim_lorenz(np.tile([2.0, 0.1], (2, 1)), n_timestep=5, phi=1.5, want_data=True)
    assert np.isnan(X.cpu().numpy()[:, 1:]).all() and np.isnan(S.cpu().numpy()).all()


def test_device_model_runs_rejection_and_smc(lorenz_double):
    import elfi_b200 as elfi
    from elfi_b200.examples import lorenz
    m, dp = lorenz.get_device_model(seed_obs=3)
    host_m = lorenz.get_model(seed_obs=3)
    assert np.array_equal(m.observed['Lorenz'], host_m.observed['Lorenz'])
    assert dp.parameter_names == ['theta1', 'theta2']
    assert dp.kinds == ['uniform', 'uniform']
    assert sorted(n for n in m.nodes if not n.startswith('_')) == sorted(
        n for n in host_m.nodes if not n.startswith('_'))
    res = elfi.Rejection(m['d'], batch_size=50, seed=1).sample(5, quantile=0.1, bar=False)
    assert res.n_samples == 5 and not np.any(np.isnan(res.discrepancies))
    smc = elfi.SMC(m['d'], batch_size=50, seed=2, device_proposal=dp).sample(
        5, quantiles=[0.5, 0.5], bar=False)
    assert len(smc.populations) == 2
    assert 'elfi_b200_sim_lorenz_f64' in lorenz_double.CALLS
