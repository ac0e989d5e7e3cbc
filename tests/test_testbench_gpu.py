"""Testbench on the H100: the segmented distance and top-n merge against R separate calls of the
one-segment entry points, bit for bit; the reference's golden testbench on the host MA2 model; and
lock-step against serial on host and device models."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from conftest import load_golden  # noqa: E402

import elfi_b200 as elfi  # noqa: E402
from elfi_b200 import device as dev  # noqa: E402
from elfi_b200 import ops  # noqa: E402
from elfi_b200.examples import ar1 as exar1  # noqa: E402
from elfi_b200.examples import ma2 as exma2  # noqa: E402

CASE = dict(seed_obs=4, repetitions=3, seed=156)
METHODS = [
    ('Rejection', dict(discrepancy_name='d', batch_size=500), dict(n_samples=500)),
    ('Rejection', dict(discrepancy_name='d', batch_size=500), dict(n_samples=100, n_sim=2000)),
    ('Rejection', dict(discrepancy_name='d', batch_size=500), dict(n_samples=50, threshold=0.5)),
    ('SMC', dict(discrepancy_name='d', batch_size=500), dict(n_samples=100,
                                                            thresholds=[2.0, 1.0])),
]


def _bits(t):
    return t.cpu().numpy().view(np.uint64)


# -- dist_seg ------------------------------------------------------------------------------------
@pytest.mark.parametrize('R', [1, 2, 7, 64])
@pytest.mark.parametrize('D,B', [(2, 1000), (16, 45), (35, 1003), (128, 77)])
@pytest.mark.parametrize('strided', [False, True])
def test_dist_seg_equals_per_segment_dist_euclid(R, D, B, strided):
    g = torch.Generator(device='cuda').manual_seed(R * 1000 + D)
    pad = 16 if strided else 0
    S = torch.randn(R * B, D + pad, dtype=torch.float64, device='cuda', generator=g)[:, :D]
    obs = torch.randn(R, D + 3 * bool(strided), dtype=torch.float64, device='cuda',
                      generator=g)[:, :D]
    S[0, 0] = float('nan')
    S[-1, -1] = float('inf')
    d = ops.dist_seg(S, obs)
    want = torch.cat([ops.dist_euclid(S[r * B:(r + 1) * B], obs[r])[0] for r in range(R)])
    assert np.array_equal(_bits(d), _bits(want))


@pytest.mark.parametrize('metric,p', [('sqeuclidean', 2.0), ('cityblock', 2.0),
                                      ('chebyshev', 2.0), ('minkowski', 3.0)])
@pytest.mark.parametrize('D', [3, 40])
def test_dist_seg_other_metrics_equal_dist_metric(metric, p, D):
    R, B = 7, 301
    g = torch.Generator(device='cuda').manual_seed(D)
    S = torch.randn(R * B, D, dtype=torch.float64, device='cuda', generator=g)
    obs = torch.randn(R, D, dtype=torch.float64, device='cuda', generator=g)
    d = ops.dist_seg(S, obs, metric, p)
    want = torch.cat([ops.dist_metric(S[r * B:(r + 1) * B], obs[r], metric, p=p)[0]
                      for r in range(R)])
    assert np.array_equal(_bits(d), _bits(want))


# -- topn_merge_seg ------------------------------------------------------------------------------
@pytest.mark.parametrize('R', [1, 3, 300])
@pytest.mark.parametrize('nA,nB,n_keep', [(0, 50, 20), (40, 70, 40), (40, 70, 110), (1, 1, 1)])
def test_topn_merge_seg_equals_separate_merges(R, nA, nB, n_keep):
    rng = np.random.RandomState(R + nA + nB)
    ka = np.round(rng.rand(R, nA) * 8) / 8          # many ties
    kb = np.round(rng.rand(R, nB) * 8) / 8
    for r in range(0, R, 2):
        kb[r, rng.randint(nB)] = np.nan
        kb[r, rng.randint(nB)] = np.inf
        kb[r, rng.randint(nB)] = -np.inf
        if nA:
            ka[r, rng.randint(nA)] = np.nan
    shapes = [(), (3,), (2, 5)]
    A = [dev.to_device(rng.randn(R, nA, *s)) for s in shapes]
    Bs = [dev.to_device(rng.randn(R, nB, *s)) for s in shapes]
    # the keys as a strided column of a (R, rows, 2) distance matrix
    KA = dev.to_device(np.stack([rng.randn(R, nA), ka], axis=2))
    KB = dev.to_device(np.stack([rng.randn(R, nB), kb], axis=2))
    tops = ops.merge_topn_seg(A, Bs, KA[:, :, 1], KB[:, :, 1], n_keep)
    for r in range(R):
        want = ops.merge_topn([a[r] for a in A], [b[r] for b in Bs], KA[r, :, 1], KB[r, :, 1],
                              None, n_keep)
        for t, w in zip(tops, want):
            assert t.shape[1:] == w.shape
            assert np.array_equal(_bits(t[r].contiguous()), _bits(w.contiguous()))


# -- the reference's golden testbench ------------------------------------------------------------
def _golden_bench():
    m = exma2.get_model(seed_obs=CASE['seed_obs'])
    tb = elfi.Testbench(model=m, repetitions=CASE['repetitions'], seed=CASE['seed'],
                        progress_bar=False)
    for k, (cls, mk, sk) in enumerate(METHODS):
        method = elfi.TestbenchMethod(method=getattr(elfi, cls), name='m{}'.format(k))
        method.set_method_kwargs(**mk)
        method.set_sample_kwargs(bar=False, **sk)
        tb.add_method(method)
    return tb


@pytest.mark.parametrize('lockstep', [True, False])
def test_golden_testbench_host_ma2(lockstep):
    g = load_golden('testbench')
    tb = _golden_bench()
    tb.run(lockstep=lockstep)
    for k, res in enumerate(tb.testbench_results):
        for r, s in enumerate(res['results']):
            key = 'sim_m{}_r{}_'.format(k, r)
            assert s.n_sim == int(g[key + 'nsim'])
            for t in ('t1', 't2'):
                if k < 3:
                    assert np.array_equal(s.samples[t], g[key + t]), (k, r, t)
                else:       # the SMC parity bar of tests/test_samplers_gpu.py
                    np.testing.assert_allclose(s.samples[t], g[key + t], rtol=1e-6, atol=1e-9)
            if k < 3:
                assert np.array_equal(s.discrepancies, g[key + 'd'])
            else:
                np.testing.assert_allclose(s.discrepancies, g[key + 'd'], rtol=1e-6, atol=1e-9)
    smd = tb.parameterwise_sample_mean_differences()
    for k in range(4):
        for t in ('t1', 't2'):
            np.testing.assert_allclose(smd['m{}'.format(k)][t], g['sim_m{}_smd_{}'.format(k, t)],
                                       rtol=0 if k < 3 else 1e-6, atol=0 if k < 3 else 1e-9)


# -- lock-step against serial --------------------------------------------------------------------
def _run(model, mk, sk, lockstep, reps, seed):
    tb = elfi.Testbench(model=model, repetitions=reps, seed=seed, progress_bar=False)
    m = elfi.TestbenchMethod(method=elfi.Rejection)
    m.set_method_kwargs(**mk)
    m.set_sample_kwargs(bar=False, **sk)
    tb.add_method(m)
    tb.run(lockstep=lockstep)
    return tb.testbench_results[0]['results']


def _same(a, b):
    for s, t in zip(a, b):
        assert list(s.outputs) == list(t.outputs)
        for k in s.outputs:
            x, y = np.asarray(s.outputs[k]), np.asarray(t.outputs[k])
            assert x.shape == y.shape and np.array_equal(x.view(np.uint64), y.view(np.uint64)), k
        for key in ('n_sim', 'n_batches', 'threshold', 'accept_rate', 'seed'):
            assert getattr(s, key) == getattr(t, key), key


@pytest.mark.parametrize('kind', ['host_ma2', 'device_ma2', 'device_ar1'])
@pytest.mark.parametrize('sk', [dict(n_samples=200, quantile=0.01),
                                dict(n_samples=50, n_sim=30000)])
def test_lockstep_equals_serial(kind, sk):
    if kind == 'host_ma2':
        m, outs, bs = exma2.get_model(seed_obs=4), ['S1', 'S2'], 2000
    elif kind == 'device_ma2':
        m, outs, bs = exma2.get_device_model(seed_obs=4), ['S1', 'S2'], 10000
    else:
        m, outs, bs = exar1.get_device_model(seed_obs=4)[0], [], 10000
    mk = dict(discrepancy_name='d', batch_size=bs, output_names=outs)
    lock = _run(m, mk, sk, True, 5, 21)
    serial = _run(m, mk, sk, False, 5, 21)
    assert len(lock) == len(serial) == 5
    _same(lock, serial)
