"""CPU checks of the g-and-k robust / octile summaries and the bivariate g-and-k example.

* elfi_b200/csrc/gnkstats.cuh built for the host (tests/harness/gnkstats_harness.cpp) against
  np.percentile and the reference's ss_robust / ss_octile restated with NumPy, bit for bit, for
  every series length 1..600, 1000 and 2048, with ties, constant rows, infinities and NaN;
* the host path of elfi_b200.examples.gnk / bignk against the golden fixtures of the unmodified
  reference (tests/golden/gen_golden_bignk.py);
* the Python layer (validation, dispatch, the throughput-mode graphs) and the samplers on the CPU
  test double extended by tests/gnk_double.py.
"""
import ctypes
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
    so = str(tmp_path_factory.mktemp('gnkstats') / 'gnkstats_harness.so')
    subprocess.check_call([gxx, '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-o', so,
                           os.path.join(HERE, 'harness', 'gnkstats_harness.cpp')])
    return ctypes.CDLL(so)


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _harness_summaries(harness, y, kind):
    """(B, n, d) -> (B, width * d, 1) through gnkstats.cuh, laid out as np.hstack."""
    from elfi_b200 import ops
    B, n, d = y.shape
    series = np.ascontiguousarray(np.sort(np.moveaxis(y, 2, 1).reshape(B * d, n), axis=1))
    w = ops.GNK_WIDTH[kind]
    out = np.empty((B * d, w))
    harness.harness_gnk_summary(_ptr(series), ctypes.c_int64(B * d), ctypes.c_int64(n),
                                ctypes.c_int32(ops.GNK_KINDS[kind]), _ptr(ops.gnk_picks(n)), _ptr(out))
    return np.moveaxis(out.reshape(B, d, w), 1, 2).reshape(B, w * d, 1)


def _rows(n, rs):
    """Series of length n: normal, heavy ties, constant (ss_B = 0), +-inf at the top / bottom (an
    infinity at a picked position, with t = 0 wherever (n - 1) q is whole), scattered infinities,
    a NaN."""
    rows = [rs.randn(n), np.round(rs.randn(n)), np.full(n, -2.5), rs.randn(n), rs.randn(n),
            rs.randn(n), rs.randn(n)]
    top = np.argsort(rows[3])
    rows[3][top[-max(1, n // 4):]] = np.inf
    rows[4][top[:max(1, n // 3)]] = -np.inf
    rows[5][rs.rand(n) < 0.3] = np.inf
    rows[5][rs.rand(n) < 0.3] = -np.inf
    rows[6][rs.randint(n)] = np.nan
    return np.stack(rows)


def _reference(y, kind):
    from elfi_b200.examples import gnk
    with np.errstate(invalid='ignore'):
        return (gnk.ss_robust if kind == 'ss_robust' else gnk.ss_octile)(y)


@pytest.mark.parametrize('d', [1, 2])
def test_header_matches_numpy_every_length(harness, d):
    rs = np.random.RandomState(d)
    for n in list(range(1, 601)) + [1000, 2048]:
        y = np.stack([_rows(n, rs) for _ in range(d)], axis=2)
        for kind in ('ss_robust', 'ss_octile'):
            got = _harness_summaries(harness, y, kind)
            want = _reference(y, kind)
            assert np.array_equal(got, want, equal_nan=True), (n, d, kind, got[:, :, 0], want[:, :, 0])


def test_octiles_are_np_percentile(harness):
    """The picks reproduce np.percentile itself (not only the restated summaries)."""
    rs = np.random.RandomState(5)
    for n in (1, 2, 3, 8, 9, 17, 50, 511, 2048):
        y = _rows(n, rs)[:, :, None]
        with np.errstate(invalid='ignore'):
            want = np.moveaxis(np.percentile(y, np.linspace(12.5, 87.5, 7), axis=1), 0, 1)
        got = _harness_summaries(harness, y, 'ss_octile')
        assert np.array_equal(got, want, equal_nan=True), n


def test_host_summaries_match_reference_golden():
    from elfi_b200.examples import gnk
    g = load_golden('bignk_summaries')
    for name in ('bignk', 'gnk', 'edge7', 'edge50', 'edge1', 'edge2'):
        y = g[name + '_y']
        with np.errstate(invalid='ignore'):
            r, o = gnk.ss_robust(y), gnk.ss_octile(y)
        assert np.array_equal(r, g[name + '_robust'], equal_nan=True), name
        assert np.array_equal(o, g[name + '_octile'], equal_nan=True), name
        assert np.array_equal(gnk.euclidean_multiss(r, observed=[r[:1]]), g[name + '_d_robust'],
                              equal_nan=True), name
        assert np.array_equal(gnk.euclidean_multiss(o, observed=[o[-1:]]), g[name + '_d_octile'],
                              equal_nan=True), name


def test_bignk_draws_match_reference_golden():
    from elfi_b200.examples import bignk, gnk
    g = load_golden('bignk_draws')
    y = bignk.BiGNK(*g['prm'], n_obs=40, batch_size=4, random_state=np.random.RandomState(3))
    assert np.array_equal(y, g['bignk_y'])
    y1 = gnk.GNK(*g['gnk_prm'], n_obs=33, batch_size=3, random_state=np.random.RandomState(4))
    assert np.array_equal(y1, g['gnk_y'])


def test_bignk_rejection_matches_reference_golden(cpu_double):
    """Rejection on bignk.get_model (host simulator and summaries) reproduces the reference's
    sample; the threshold and the selection run through the (CPU double of the) device kernels."""
    import elfi_b200 as elfi
    from elfi_b200.examples import bignk
    g = load_golden('bignk_rejection')
    m = bignk.get_model(seed=11)
    assert np.array_equal(m.observed['BiGNK'], g['observed_BiGNK'])
    res = elfi.Rejection(m['d'], batch_size=10, seed=5).sample(20, bar=False)
    assert res.n_sim == int(g['n_sim'])
    assert res.threshold == float(g['threshold'])
    assert np.array_equal(res.discrepancies, g['out_d'])
    for name in bignk.PARAMETER_NAMES:
        assert np.array_equal(res.samples[name], g['out_' + name]), name


@pytest.fixture
def gnk_double(cpu_double, monkeypatch):
    import abi_double
    import gnk_double
    import priors_double
    abi_double.install(monkeypatch, priors_double.TABLE, gnk_double.TABLE)
    return cpu_double


def test_picks_follow_numpy_indexing():
    from elfi_b200 import ops
    p = ops.gnk_picks(1)
    assert np.array_equal(p, [0] * 14 + [1.0] * 7)     # vi >= n - 1: the last element, t = vi + 1
    p = ops.gnk_picks(9)
    assert np.array_equal(p[:7], np.arange(1, 8)) and np.array_equal(p[14:], np.zeros(7))
    p = ops.gnk_picks(150)
    assert np.array_equal(p[7:14], p[:7] + 1) and np.all((p[14:] >= 0) & (p[14:] < 1))


def test_ops_validate_before_the_call(gnk_double):
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    with pytest.raises(ValueError, match='2048'):
        ops.gnk_summaries(np.zeros((2, 2049, 1)))
    with pytest.raises(ValueError, match='1 or 2'):
        ops.gnk_summaries(np.zeros((2, 10, 3)))
    with pytest.raises(ValueError, match='unknown'):
        ops.gnk_summaries(np.zeros((2, 10, 1)), kind='ss_order')
    with pytest.raises(ValueError, match='512'):
        ops.sim_gnk_summaries(*[np.ones(3)] * 4, n_obs=513)
    with pytest.raises(ValueError, match='512'):
        ops.sim_bignk(np.ones((3, 9)), n_obs=513, kind='ss_robust')
    with pytest.raises(ValueError, match='9 parameters'):
        ops.sim_bignk(np.ones((3, 8)))
    with pytest.raises(ValueError, match='128'):
        ops.euclidean_multiss(dev.to_device(np.zeros((2, 129))), np.zeros(129))
    assert not gnk_double.CALLS


def test_dispatch_host_device_and_lazy_agree(gnk_double):
    """ss_robust / ss_octile / euclidean_multiss on host arrays, device tensors (strided views
    included) and lazy simulator output give the same values."""
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    from elfi_b200.examples import bignk, gnk
    rs = np.random.RandomState(0)
    y = rs.randn(5, 37, 2)
    big = dev.to_device(np.concatenate([y, rs.randn(5, 3, 2)], axis=1))
    for fn in (gnk.ss_robust, gnk.ss_octile):
        host = fn(y)
        devv = fn(big[:, :37, :])
        assert devv.shape == host.shape and np.array_equal(devv.cpu().numpy(), host)
        d_host = gnk.euclidean_multiss(host, observed=[host[:1]])
        d_dev = gnk.euclidean_multiss(devv, observed=[host[:1]])
        assert np.array_equal(d_dev.cpu().numpy(), d_host)
    lazy = gnk.gnk_device_lazy(3, 1, 2, .5, n_obs=40, batch_size=6, random_state=np.random.RandomState(1))
    data = lazy.materialize()
    assert tuple(data.shape) == (6, 40, 1)
    assert np.array_equal(gnk.ss_robust(lazy).cpu().numpy(), gnk.ss_robust(data.cpu().numpy()))
    lazy2 = bignk.bignk_device(*[1.0] * 8, 0.5, n_obs=30,
                               batch_size=4, random_state=np.random.RandomState(2))
    data2 = lazy2.materialize()
    assert tuple(data2.shape) == (4, 30, 2)
    assert np.array_equal(gnk.ss_octile(lazy2).cpu().numpy(), gnk.ss_octile(data2.cpu().numpy()))
    Y, S = ops.sim_bignk(np.tile([1, 2, 1, 1, 0, 0, 0, 0, 2.0], (3, 1)), n_obs=10, kind='ss_robust')
    assert np.isnan(Y.cpu().numpy()).all() and np.isnan(S.cpu().numpy()).all()   # |rho| > 1


def test_device_models_run_rejection_and_smc(gnk_double):
    import elfi_b200 as elfi
    from elfi_b200.examples import bignk, gnk
    m, dp = bignk.get_device_model(n_obs=60, seed=3)
    assert dp.parameter_names == bignk.PARAMETER_NAMES
    res = elfi.Rejection(m['d'], batch_size=500, seed=1).sample(50, quantile=0.1, bar=False)
    assert res.n_samples == 50 and np.all(np.isfinite(res.discrepancies))
    smc = elfi.SMC(m['d'], batch_size=500, seed=2, device_proposal=dp).sample(
        50, thresholds=[np.inf, np.inf], bar=False)
    assert len(smc.populations) == 2
    for kind in ('ss_robust', 'ss_octile'):
        mg, prop = gnk.get_device_model(n_obs=50, seed=3, summary=kind)
        res = elfi.Rejection(mg['d'], batch_size=400, seed=1).sample(40, quantile=0.1, bar=False)
        assert res.n_samples == 40 and np.all(np.isfinite(res.discrepancies))
        smc = elfi.SMC(mg['d'], batch_size=400, seed=2, device_proposal=prop).sample(
            40, quantiles=[0.5, 0.5], bar=False)
        assert len(smc.populations) == 2
    assert 'elfi_b200_sim_bignk_f64' in gnk_double.CALLS
    assert 'elfi_b200_sim_gnk_summaries_f64' in gnk_double.CALLS
    assert 'elfi_b200_euclidean_multiss_f64' in gnk_double.CALLS
    with pytest.raises(ValueError, match='summary'):
        gnk.get_device_model(summary='ss_order')
