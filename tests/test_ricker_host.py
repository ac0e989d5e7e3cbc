"""CPU checks of the Ricker example and the Poisson sampler.

* the host path of elfi_b200.examples.ricker against the golden fixtures of the unmodified reference
  (tests/golden/gen_golden_ricker.py), bit for bit: draws, summaries, chi_squared, Rejection;
* elfi_b200/csrc/poisson.cuh built for the host (tests/harness/poisson_harness.cpp): its log-pmf
  against mpmath at 50 digits, and its accept / reject decisions against the NumPy replay
  tests/ricker_replay.py;
* the Python layer (validation, dispatch, the throughput-mode graphs) and the samplers on the CPU
  test double extended by tests/ricker_double.py.
"""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

import ricker_replay as rr
from conftest import load_golden

HERE = os.path.dirname(os.path.abspath(__file__))
# |log-pmf - mpmath| for rates 10 .. 9.2e18 and k within 10 sd: the terms of Loader's form are all
# below ~50, so a few 1e-14 is what double precision allows
LOGPMF_ABS_BOUND = 1e-12


@pytest.fixture(scope='module')
def harness(tmp_path_factory):
    gxx = shutil.which('g++')
    if gxx is None:
        pytest.skip('g++ not available')
    so = str(tmp_path_factory.mktemp('poisson') / 'poisson_harness.so')
    subprocess.check_call([gxx, '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-o', so,
                           os.path.join(HERE, 'harness', 'poisson_harness.cpp')])
    return ctypes.CDLL(so)


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _logpmf(harness, k, lam):
    k = np.ascontiguousarray(k, dtype=np.float64)
    lam = np.ascontiguousarray(np.broadcast_to(lam, k.shape), dtype=np.float64)
    out = np.empty_like(k)
    harness.harness_poisson_logpmf(_ptr(k), _ptr(lam), ctypes.c_int64(k.size), _ptr(out))
    return out


def _draw(harness, lam, rows, seed, base, salt):
    lam = np.ascontiguousarray(lam, dtype=np.float64)
    rows = np.ascontiguousarray(rows, dtype=np.uint64)
    k, margin = np.empty_like(lam), np.empty_like(lam)
    trials = np.empty(lam.shape, dtype=np.int32)
    harness.harness_poisson_draw(_ptr(lam), _ptr(rows), ctypes.c_int64(lam.size), ctypes.c_uint64(seed),
                                 ctypes.c_uint32(base), ctypes.c_uint32(salt), _ptr(k), _ptr(trials),
                                 _ptr(margin))
    return k, trials, margin


def _mp_logpmf(k, lam):
    import mpmath as mp
    with mp.workdps(50):
        k, lam = mp.mpf(float(k)), mp.mpf(float(lam))
        return -lam + k * mp.log(lam) - mp.loggamma(k + 1)


def _grid():
    """(k, lam, exact) for rates 10 .. 9.2e18 and k within +-10 sd."""
    ks, lams, exact = [], [], []
    for lam in np.concatenate([np.geomspace(10, 9.2e18, 24), [1e14]]):
        sd = np.sqrt(lam)
        for z in np.linspace(-10, 10, 21):
            k = np.floor(lam + z * sd)
            if k < 0:
                continue
            ks.append(k)
            lams.append(lam)
            exact.append(_mp_logpmf(k, lam))
    return np.array(ks), np.array(lams), exact


def test_logpmf_matches_mpmath_where_numpys_form_fails(harness):
    k, lam, exact = _grid()
    got = _logpmf(harness, k, lam)
    err = np.array([float(abs(g - e)) for g, e in zip(got, exact)])
    assert err.max() < LOGPMF_ABS_BOUND, (err.max(), k[err.argmax()], lam[err.argmax()])
    replay = rr.logpmf(k, lam)
    assert np.max(np.abs(replay - got)) < LOGPMF_ABS_BOUND
    at14 = lam == 1e14
    numpy_form = rr.logpmf_numpy_form(k[at14], lam[at14])
    err14 = np.array([float(abs(g - e)) for g, e in zip(numpy_form, np.array(exact, dtype=object)[at14])])
    assert err14.max() > 1e3 * LOGPMF_ABS_BOUND, err14.max()


def test_stirlerr_table_and_series_meet(harness):
    """At k = 15 / 16 the table hands over to the series: both agree with mpmath."""
    for k in (1.0, 2.0, 15.0, 16.0, 17.0, 40.0):
        got = _logpmf(harness, np.array([k]), 12.5)[0]
        assert abs(got - float(_mp_logpmf(k, 12.5))) < 1e-14, k


def test_edge_rates(harness):
    lam = np.array([0.0, -1.0, np.nan, np.inf, rr.LAM_MAX, np.nextafter(rr.LAM_MAX, np.inf), 1e-300])
    k, trials, _ = _draw(harness, lam, np.arange(lam.size), 5, 0, rr.SALT_POISSON)
    assert k[0] == 0 and trials[0] == 0
    assert np.isnan(k[1:4]).all() and np.isnan(k[5])
    assert np.isfinite(k[4]) and abs(k[4] - rr.LAM_MAX) < 2e10
    assert k[6] == 0


def test_decisions_equal_the_replay(harness):
    """Host build and NumPy replay draw the same counts, apart from knife-edge decisions (a margin
    below rr.POISSON_MARGIN), which are excluded and counted."""
    rates = [1e-3, 0.5, 5, 9.999, 10, 10.5, 37, 1e3, 1e6, 1e12, 1e15, 1e18]
    n = 20000
    excluded = 0
    for i, lam0 in enumerate(rates):
        lam = np.full(n, float(lam0))
        rows = np.arange(n, dtype=np.uint64) + np.uint64(2 ** 32 - n // 2)
        k, trials, margin = _draw(harness, lam, rows, 17 + i, 0, rr.SALT_POISSON)
        rk, rtrials, rmargin, kind = rr.draw(lam, rows, 17 + i, 0, rr.SALT_POISSON)
        amb = rr.ambiguous(np.minimum(margin, rmargin), kind)
        excluded += int(amb.sum())
        assert np.array_equal(k[~amb], rk[~amb]), lam0
        assert np.array_equal(trials[~amb], rtrials[~amb]), lam0
        assert np.allclose(margin[~amb], rmargin[~amb], rtol=1e-6, atol=1e-11)
    assert excluded <= 5, excluded


# ---------------------------------------------------------------------------- reference goldens
def test_host_draws_match_reference_golden():
    from elfi_b200.examples import ricker
    g = load_golden('ricker_draws')
    prm = g['stoch_prm']
    y = ricker.stochastic_ricker(*prm.T, n_obs=30, batch_size=len(prm),
                                 random_state=np.random.RandomState(3))
    assert np.array_equal(y, g['stoch_y'])
    assert (y == 0).all(axis=1).sum() == 0 and (y == 0).sum() > 0 and y.max() > 1e9
    r = g['det_rates']
    assert np.array_equal(ricker.ricker(r, n_obs=40, batch_size=len(r)), g['det_y1'])
    assert np.array_equal(ricker.ricker(r, stock_init=0.25, n_obs=40, batch_size=len(r)), g['det_y2'])


def test_host_summaries_and_chi_squared_match_reference_golden():
    from elfi_b200.examples import ricker
    g = load_golden('ricker_summaries')
    draws = load_golden('ricker_draws')
    for name, y in (('stoch', draws['stoch_y']), ('det', draws['det_y1'])):
        s = (ricker.ss_mean(y), ricker.ss_var(y), ricker.num_zeros(y))
        for v, key in zip(s, ('_mean', '_var', '_zeros')):
            assert np.array_equal(v, g[name + key]), name + key
        for tag in ('row0', 'nozero', 'mostzeros', 'extinct'):
            o = g['{}_obs_{}'.format(name, tag)]
            with np.errstate(divide='ignore', invalid='ignore'):
                chi = ricker.chi_squared(*s, observed=tuple(o[:, None]))
            assert np.array_equal(chi, g['{}_chi_{}'.format(name, tag)], equal_nan=True), (name, tag)
    assert np.isnan(g['stoch_chi_nozero']).any() and np.isinf(g['stoch_chi_extinct']).all()


@pytest.mark.parametrize('variant', ['stochastic', 'deterministic'])
def test_rejection_matches_reference_golden(cpu_double, variant):
    """Rejection on get_model (host simulator and summaries) reproduces the reference's sample."""
    import elfi_b200 as elfi
    from elfi_b200.examples import ricker
    g = load_golden('ricker_rejection')
    m = ricker.get_model(seed_obs=7, stochastic=variant == 'stochastic')
    assert np.array_equal(m.observed['Ricker'], g[variant + '_observed'])
    res = elfi.Rejection(m['d'], batch_size=20, seed=3).sample(30, bar=False)
    assert res.n_sim == int(g[variant + '_n_sim'])
    assert res.threshold == float(g[variant + '_threshold'])
    assert np.array_equal(res.discrepancies, g[variant + '_d'])
    names = ['t1', 't2', 't3'] if variant == 'stochastic' else ['t1']
    for name in names:
        assert np.array_equal(res.samples[name], g['{}_out_{}'.format(variant, name)]), name


# ---------------------------------------------------------------------------- Python layer
@pytest.fixture
def ricker_double(cpu_double, monkeypatch):
    import abi_double
    import priors_double
    import ricker_double
    abi_double.install(monkeypatch, priors_double.TABLE, ricker_double.TABLE)
    return cpu_double


def test_ops_validate_before_the_call(ricker_double):
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    with pytest.raises(ValueError, match='stock_init'):
        ops.sim_ricker(np.ones((2, 3)), stock_init=np.ones(2))
    with pytest.raises(ValueError, match='n_obs'):
        ops.sim_ricker(np.ones((2, 3)), n_obs=0)
    with pytest.raises(ValueError, match='3 parameters'):
        ops.sim_ricker(np.ones((2, 2)))
    with pytest.raises(ValueError, match='1 parameter'):
        ops.sim_ricker(np.ones((2, 3)), stochastic=False)
    with pytest.raises(ValueError, match='128'):
        ops.chi_squared(dev.to_device(np.ones((2, 129))), np.ones(129))
    with pytest.raises(ValueError, match='values'):
        ops.chi_squared(dev.to_device(np.ones((2, 3))), np.ones(2))
    assert not ricker_double.CALLS


def test_dispatch_host_device_and_lazy_agree(ricker_double):
    """ss_mean / ss_var / num_zeros / chi_squared on host arrays, device tensors and lazy simulator
    output give the same values; above the fused cap the lazy data is written and summarised."""
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    from elfi_b200.examples import ricker
    rs = np.random.RandomState(0)
    y = rs.poisson(rs.choice([0.0, 0.5, 20.0], size=(7, 1)), size=(7, 30)).astype(float)
    fns = (ricker.ss_mean, ricker.ss_var, ricker.num_zeros)
    host = [f(y) for f in fns]
    devv = [f(dev.to_device(y)) for f in fns]
    for h, d_ in zip(host, devv):
        assert np.array_equal(d_.cpu().numpy(), h)
    S = ops.ricker_summaries(y)
    assert np.array_equal(S.cpu().numpy(), np.stack(host, axis=1))
    obs = tuple(np.array([v[0] if i < 2 else 0.0]) for i, v in enumerate(host))
    with np.errstate(divide='ignore', invalid='ignore'):
        chi_h = ricker.chi_squared(*host, observed=obs)
        chi_d = ricker.chi_squared(*devv, observed=obs)
    assert np.array_equal(chi_d.cpu().numpy(), chi_h, equal_nan=True)
    for n_obs in (40, ops.RICKER_FUSED_MAX + 1):
        for stochastic, params in ((True, (3.8, 0.3, 10)), (False, (3.8,))):
            lazy = ricker.ricker_device(*params, n_obs=n_obs, stochastic=stochastic, batch_size=5,
                                        random_state=np.random.RandomState(1))
            data = lazy.materialize()
            assert tuple(data.shape) == (5, n_obs)
            for f in fns:
                assert np.array_equal(f(lazy).cpu().numpy(), f(data.cpu().numpy())), (f, n_obs)
    nan_rows = ops.sim_ricker(np.tile([3.8, 0.3, -1.0], (3, 1)), n_obs=5, want_data=True)
    assert np.isnan(nan_rows[0].cpu().numpy()).all()     # negative rates: NaN counts


@pytest.mark.parametrize('stochastic', [True, False])
def test_device_models_run_rejection_and_smc(ricker_double, stochastic):
    import elfi_b200 as elfi
    from elfi_b200.examples import ricker
    m, dp = ricker.get_device_model(seed_obs=3, stochastic=stochastic)
    assert dp.parameter_names == (['t1', 't2', 't3'] if stochastic else ['t1'])
    assert dp.kinds == (['expon', 'truncnorm', 'uniform'] if stochastic else ['expon'])
    res = elfi.Rejection(m['d'], batch_size=500, seed=1).sample(50, quantile=0.1, bar=False)
    assert res.n_samples == 50 and not np.any(np.isnan(res.discrepancies))
    smc = elfi.SMC(m['d'], batch_size=500, seed=2, device_proposal=dp).sample(
        50, quantiles=[0.5, 0.5], bar=False)
    assert len(smc.populations) == 2
    assert 'elfi_b200_sim_ricker_f64' in ricker_double.CALLS
    if stochastic:
        assert 'elfi_b200_chi_squared_f64' in ricker_double.CALLS
    with pytest.raises(ValueError, match='n_obs'):
        ricker.get_device_model(n_obs=0)
