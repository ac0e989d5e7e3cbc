"""CPU checks of the AR(1) example and of compare_models.

* the host path of elfi_b200.examples.ar1 against the golden fixtures of the unmodified reference
  (tests/golden/gen_golden_ar1.py), bit for bit: draws and Rejection;
* elfi_b200/csrc/ar1.cuh built for the host (tests/harness/ar1_harness.cpp, -ffp-contract=off): the
  step fed the reference's normals gives its series, and the fused distance equals SciPy's cdist;
* the Python layer on the CPU test double extended by tests/ar1_double.py: validation, the lazy
  output, and a Euclidean Distance taking the fused or the materialised path;
* compare_models against the reference's result on the golden discrepancies, and its errors.
"""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
from scipy.spatial.distance import cdist

from conftest import load_golden

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope='module')
def harness(tmp_path_factory):
    gxx = shutil.which('g++')
    if gxx is None:
        pytest.skip('g++ not available')
    so = str(tmp_path_factory.mktemp('ar1') / 'ar1_harness.so')
    subprocess.check_call([gxx, '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-o',
                           so, os.path.join(HERE, 'harness', 'ar1_harness.cpp')])
    return ctypes.CDLL(so)


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _rows(harness, phi, w, y=None):
    phi = np.ascontiguousarray(phi, dtype=np.float64)
    w = np.ascontiguousarray(w, dtype=np.float64)
    B, n = w.shape
    X = np.empty((B, n))
    d = np.empty(B) if y is not None else None
    harness.harness_ar1_rows(_ptr(phi), _ptr(w), ctypes.c_int64(B), ctypes.c_int32(n),
                             None if y is None else _ptr(np.ascontiguousarray(y, np.float64)),
                             _ptr(X), None if d is None else _ptr(d))
    return X, d


def _same_bits(a, b):
    """Equal values, NaN where NaN, and the same sign of every zero."""
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True) and \
        np.array_equal(np.signbit(a[a == 0]), np.signbit(b[a == 0]))


class _GivenRandn:
    """A RandomState stand-in whose randn hands out a given array."""

    def __init__(self, w):
        self.w = w

    def randn(self, *shape):
        assert shape == self.w.shape
        return self.w


# ---------------------------------------------------------------------------- reference goldens
def test_host_draws_match_reference_golden():
    from elfi_b200.examples import ar1
    g = load_golden('ar1_draws')
    n_keys = 0
    for j, phi in enumerate(g['phis']):
        for n in (1, 2, 200):
            for b in (1, 16):
                rs = np.random.RandomState(100 * j + 10 * n + b)
                x = ar1.AR1(phi, n_obs=n, batch_size=b, random_state=rs)
                assert _same_bits(x, g['phi{}_n{}_b{}'.format(j, n, b)]), (phi, n, b)
                n_keys += 1
    assert n_keys == 30


@pytest.mark.parametrize('tag,a', [('test', dict(seed_obs=4, batch_size=10, seed=5, n=10,
                                                 quantile=0.5)),
                                   ('q', dict(seed_obs=1, batch_size=100, seed=3, n=50,
                                              quantile=0.1))])
def test_rejection_matches_reference_golden(cpu_double, tag, a):
    import elfi_b200 as elfi
    from elfi_b200.examples import ar1
    g = load_golden('ar1_rejection')
    m = ar1.get_model(seed_obs=a['seed_obs'])
    assert _same_bits(m.observed['AR1'], g[tag + '_observed'])
    res = elfi.Rejection(m['d'], batch_size=a['batch_size'], seed=a['seed']).sample(
        a['n'], quantile=a['quantile'], bar=False)
    assert res.n_sim == int(g[tag + '_n_sim'])
    assert res.threshold == float(g[tag + '_threshold'])
    assert _same_bits(res.discrepancies, g[tag + '_d'])
    assert _same_bits(res.samples['phi'], g[tag + '_phi'])


def test_graph_names_match_the_reference():
    from elfi_b200.examples import ar1
    m = ar1.get_model(seed_obs=0, n_obs=20)
    assert m.parameter_names == ['phi']
    assert {'phi', 'AR1', 'd'} <= set(m.nodes)
    assert m.observed['AR1'].shape == (1, 20)
    assert _same_bits(m.observed['AR1'],
                      ar1.AR1(0.9, n_obs=20, random_state=np.random.RandomState(0)))


# ---------------------------------------------------------------------------- ar1.cuh on the host
def test_step_and_distance_equal_numpy_and_scipy(harness):
    """The header's step, fed the innovations the reference's AR1 draws, gives its series bit for
    bit, and the distance accumulated step by step is SciPy's cdist of that series."""
    from elfi_b200.examples import ar1
    rs = np.random.RandomState(7)
    for n in (1, 2, 3, 200, 1000):
        B = 300
        phi = rs.uniform(-1, 1, B)
        phi[:9] = [-1.0, -0.5, 0.0, -0.0, 0.9, 1.0, 1.5, -3.0, 1e200]
        phi[9:12] = [np.nan, np.inf, -np.inf]
        w = rs.randn(B, n + 1)
        w[12, -1] = np.inf
        w[13, 0 if n == 1 else 1] = np.nan
        w[14, 1:] = -0.0
        w[15, 1:] = 0.0
        y = rs.randn(n) * 3
        with np.errstate(all='ignore'):
            want = ar1.AR1(phi, n_obs=n, batch_size=B, random_state=_GivenRandn(w.copy()))
            X, d = _rows(harness, phi, w[:, 1:], y)
            want_d = cdist(want, y[None, :], 'euclidean')[:, 0]
        assert _same_bits(X, want), n
        assert _same_bits(d, want_d), n
        assert (X[14] == 0).all() and (X[15] == 0).all()     # signed zeros, compared bit for bit


# ---------------------------------------------------------------------------- Python layer
@pytest.fixture
def ar1_double(cpu_double, monkeypatch):
    import abi_double
    import ar1_double
    import priors_double
    abi_double.install(monkeypatch, priors_double.TABLE, ar1_double.TABLE)
    return cpu_double


def test_ops_validate_before_the_call(ar1_double, monkeypatch):
    from elfi_b200 import ops
    phi = np.full(4, 0.5)
    obs = np.zeros(10)
    with pytest.raises(ValueError, match='n_obs'):
        ops.sim_ar1(phi, n_obs=0)
    with pytest.raises(ValueError, match='n_obs'):
        ops.sim_ar1(phi, n_obs=ops.AR1_NOBS_MAX + 1)
    with pytest.raises(ValueError, match='n_obs'):
        ops.sim_ar1(phi, n_obs=2.5)
    with pytest.raises(ValueError, match='1 parameters'):
        ops.sim_ar1(np.ones((4, 2)), n_obs=10)
    with pytest.raises(ValueError, match='observed'):
        ops.sim_ar1(phi, n_obs=10, thresholds=1.0)
    with pytest.raises(ValueError, match='neither'):
        ops.sim_ar1(phi, n_obs=10, want_data=False)
    with pytest.raises(ValueError, match='same number of columns'):
        ops.sim_ar1(phi, n_obs=10, obs=np.zeros(9))
    with pytest.raises(ValueError, match='one threshold'):
        ops.sim_ar1(phi, n_obs=10, obs=obs, thresholds=[1.0, 2.0])
    monkeypatch.setattr(ops, 'AR1_BATCH_MAX', 3)
    with pytest.raises(ValueError, match='at most 3 rows'):
        ops.sim_ar1(phi, n_obs=10)
    assert not ar1_double.CALLS


def test_sim_ar1_outputs(ar1_double):
    """Data, distance and accepted rows of one call agree with dist_euclid of the data, for host
    and device thresholds."""
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    rs = np.random.RandomState(1)
    phi = rs.uniform(-1, 1, 50)
    obs = rs.randn(30)
    X, d, idx = ops.sim_ar1(phi, n_obs=30, seed=3)
    assert tuple(X.shape) == (50, 30) and d is None and idx is None
    d_ref, _ = ops.dist_euclid(X, obs)
    thr = float(np.median(d_ref.cpu().numpy()))
    for t in (thr, dev.to_device(np.array([thr]))):
        X2, d2, idx2 = ops.sim_ar1(phi, n_obs=30, seed=3, obs=obs, thresholds=t)
        assert X2 is None
        want_d, want_idx = ops.dist_euclid(X, obs, thresholds=t)
        assert _same_bits(d2.cpu().numpy(), want_d.cpu().numpy())
        assert np.array_equal(idx2.cpu().numpy(), want_idx.cpu().numpy())
    X3, d3, idx3 = ops.sim_ar1(phi[:, None], n_obs=30, seed=3, obs=obs, want_data=True)
    assert _same_bits(X3.cpu().numpy(), X.cpu().numpy()) and idx3 is None
    assert _same_bits(d3.cpu().numpy(), d_ref.cpu().numpy())
    _, d0, idx0 = ops.sim_ar1(np.empty(0), n_obs=30, obs=obs, thresholds=1.0)
    assert d0.shape[0] == 0 and idx0.shape[0] == 0


def test_lazy_output(ar1_double):
    from elfi_b200 import ops
    from elfi_b200.examples import ar1, ma2
    lazy = ar1.ar1_device(0.5, n_obs=30, batch_size=7, random_state=np.random.RandomState(1))
    assert lazy.shape == (7, 30) and len(lazy) == 7
    X = lazy.materialize()
    assert lazy.materialize() is X and tuple(X.shape) == (7, 30)
    with pytest.raises(ValueError, match='no fused summaries.*materialize'):
        lazy.summaries()
    with pytest.raises(ValueError, match='no fused summaries'):
        ma2.autocov(lazy)              # another example's summary cannot read foreign columns
    obs = np.linspace(-1, 1, 30)
    d, idx = lazy.euclidean(obs, 2.0)
    want_d, want_idx = ops.dist_euclid(X, obs, thresholds=2.0)
    assert _same_bits(d.cpu().numpy(), want_d.cpu().numpy())
    assert np.array_equal(idx.cpu().numpy(), want_idx.cpu().numpy())


def test_distance_takes_the_fused_or_the_materialised_path(ar1_double):
    """A Euclidean distance of the lazy output alone runs the simulator with the distance fused
    and no distance kernel; weighted, other metrics and AdaptiveDistance materialise the data."""
    import elfi_b200 as elfi
    from elfi_b200 import model as em
    from elfi_b200.examples import ar1
    calls = ar1_double.CALLS
    obs = np.linspace(-1, 1, 30)[None, :]

    def lazy():
        return ar1.ar1_device(0.5, n_obs=30, batch_size=40, random_state=np.random.RandomState(1))
    X = lazy().materialize().cpu().numpy()
    want = cdist(X, obs)[:, 0]

    del calls[:]
    out = em.device_euclidean_discrepancy(lazy(), observed=(obs,), accept=np.array([2.5]))
    assert calls == ['elfi_b200_sim_ar1_f64']
    assert _same_bits(out.value.cpu().numpy(), want)
    assert np.array_equal(out.accepted.cpu().numpy(), np.flatnonzero(want <= 2.5))

    del calls[:]
    d = em.device_euclidean_discrepancy(lazy(), observed=(obs,))
    assert calls == ['elfi_b200_sim_ar1_f64'] and _same_bits(d.cpu().numpy(), want)

    del calls[:]
    w = np.full(30, 2.0)
    d = em.device_euclidean_discrepancy(lazy(), observed=(obs,), w=w)
    assert calls == ['elfi_b200_sim_ar1_f64', 'elfi_b200_dist_euclid_thr_f64']
    assert _same_bits(d.cpu().numpy(), cdist(X, obs, w=w)[:, 0])

    del calls[:]
    d = em.device_metric_discrepancy('cityblock', lazy(), observed=(obs,))
    assert calls == ['elfi_b200_sim_ar1_f64', 'elfi_b200_dist_metric_thr_f64']
    assert _same_bits(d.cpu().numpy(), cdist(X, obs, 'cityblock')[:, 0])

    # host data (the host model) keeps the distance kernel
    del calls[:]
    d = em.device_euclidean_discrepancy(X, observed=(obs,))
    assert calls == ['elfi_b200_dist_euclid_thr_f64'] and _same_bits(d.cpu().numpy(), want)

    m = elfi.new_model()
    elfi.Prior('uniform', -1, 2, model=m, name='phi')
    elfi.Simulator(lambda phi, batch_size=1, random_state=None: lazy(), m['phi'], observed=obs,
                   name='AR1')
    ad = elfi.AdaptiveDistance(m['AR1'], name='d')
    del calls[:]
    out = m.generate(40, outputs=['d'], seed=1)['d']
    assert 'elfi_b200_sim_ar1_f64' in calls and 'elfi_b200_dist_euclid_mom_f64' in calls
    assert ad.name == 'd' and _same_bits(out.cpu().numpy().reshape(-1), want)


def test_device_model_runs_rejection_and_smc(ar1_double):
    import elfi_b200 as elfi
    from elfi_b200.examples import ar1
    m, dp = ar1.get_device_model(seed_obs=3, n_obs=40)
    assert dp.parameter_names == ['phi'] and dp.kinds == ['uniform']
    host = ar1.get_model(seed_obs=3, n_obs=40)
    assert np.array_equal(m.observed['AR1'], host.observed['AR1'])
    res = elfi.Rejection(m['d'], batch_size=500, seed=1).sample(50, quantile=0.1, bar=False)
    assert res.n_samples == 50 and not np.any(np.isnan(res.discrepancies))
    smc = elfi.SMC(m['d'], batch_size=500, seed=2, device_proposal=dp).sample(
        50, quantiles=[0.5, 0.5], bar=False)
    assert len(smc.populations) == 2
    m['d'].become(elfi.AdaptiveDistance(m['AR1']))
    ad = elfi.AdaptiveDistanceSMC(m['d'], batch_size=500, seed=3, device_proposal=dp).sample(
        50, rounds=2, quantile=0.5, bar=False)
    assert len(ad.populations) == 2
    assert 'elfi_b200_sim_ar1_f64' in ar1_double.CALLS
    with pytest.raises(ValueError, match='n_obs'):
        ar1.get_device_model(n_obs=0)


# ---------------------------------------------------------------------------- compare_models
def _golden_samples(device=False):
    import torch

    from elfi_b200.results import DeviceOutputs, Sample
    g = load_golden('compare_models')
    out = []
    for i in range(3):
        d = g['d{}'.format(i)]
        outputs = {'mu': np.zeros(len(d)), 'd': d}
        if device:
            outputs = DeviceOutputs({k: torch.from_numpy(v.copy()) for k, v in outputs.items()})
        out.append(Sample('Rejection', outputs, ['mu'], discrepancy_name='d',
                          n_sim=int(g['n_sim{}'.format(i)])))
        assert out[-1].n_samples == int(g['n_samples{}'.format(i)])
    return g, out


@pytest.mark.parametrize('device', [False, True])
def test_compare_models_matches_reference_golden(device):
    import elfi_b200 as elfi
    g, samples = _golden_samples(device)
    assert _same_bits(elfi.compare_models(samples), g['p'])
    assert _same_bits(elfi.compare_models(samples, g['model_priors']), g['p_priors'])
    assert g['p'][0] > g['p'][1] > g['p'][2]


def test_compare_models_errors():
    import elfi_b200 as elfi
    from elfi_b200.results import Sample
    _, samples = _golden_samples()
    bare = Sample('Rejection', {'mu': np.zeros(5)}, ['mu'], n_sim=10)
    with pytest.raises(ValueError, match='valid discrepancies'):
        elfi.compare_models(samples + [bare])
    with pytest.raises(ValueError):
        elfi.compare_models([])
