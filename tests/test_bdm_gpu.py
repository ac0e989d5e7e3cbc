"""Device birth-death-mutation simulator and summaries.

* per-row replay (tests/bdm_replay.py over oracle/streams.py): counts and event counts equal the
  kernel's exactly at the four law points and at N in {1, 20, 473, 1024}, for invalid rates and
  for capped rows;
* rows are pure functions of (seed, offset + i): split launches and repeated calls agree;
* the fused T1 / T2 equal ops.bdm_summaries of the written counts and NumPy's T1 / T2, bit for bit,
  for n != 20 and strided data too;
* the law against the reference executable (tests/golden/bdm_law.npz): a two-sample KS test on T1,
  the extinction fraction and the mean number of clusters;
* throughput-mode Rejection against the reference's Rejection sample, and SMC.
"""
import numpy as np
import pytest
import scipy.stats as ss

import bdm_replay
from conftest import load_golden

pytestmark = pytest.mark.gpu
LAW_POINTS = [(0.2, 0.0, 0.198, 20), (0.005, 0.0, 0.198, 20), (1.0, 0.3, 0.198, 20),
              (1.0, 0.1, 0.198, 473)]


def _np(t):
    return t.cpu().numpy()


def _host_summaries(x, n=20):
    from elfi_b200.examples import bdm
    with np.errstate(all='ignore'):
        return np.column_stack([bdm.T1(x), bdm.T2(x, n)])


def _check_replay(P, N, seed, offset=0, max_events=2 ** 24):
    from elfi_b200 import ops
    X, S, n = ops.sim_bdm(P, N, seed=seed, offset=offset, max_events=max_events)
    X, S, n = _np(X), _np(S), _np(n)
    want, kw = bdm_replay.simulate(P, N, seed, offset, max_events)
    bad = np.nonzero(~np.all(X == want, axis=1) | (n != kw))[0]
    assert bad.size == 0, (bad[:5], n[bad[:5]], kw[bad[:5]])
    return X, S, n


@pytest.mark.parametrize('point', LAW_POINTS)
def test_replay_law_points(point):
    P = np.tile(point[:3], (4096, 1))
    X, S, n = _check_replay(P, int(point[3]), seed=11, offset=2 ** 32 - 1000)
    assert np.all(n > 0)


@pytest.mark.parametrize('N', [1, 20, 473, 1024])
def test_replay_every_N_with_invalid_and_capped_rows(N):
    rs = np.random.RandomState(N)
    B = 512 if N <= 20 else 256
    P = np.column_stack([rs.uniform(0.5, 2.0, B), rs.uniform(0, 0.3, B), np.full(B, 0.198)])
    P[:6] = [(-1.0, 0, 1), (0, 0, 0), (np.nan, 0, 1), (1, np.inf, 1), (1e308, 1e308, 1e308),
             (0, 0.5, 0)]
    X, S, n = _check_replay(P, N, seed=5)
    assert np.all(n[:5] == -1) and np.all(X[:5] == -1) and np.isnan(S[:5]).all()
    assert n[5] == 1 and np.all(X[5] == 0) and np.isnan(S[5, 0])
    ok = np.all(X >= 0, axis=1)
    assert np.array_equal(S[ok], _host_summaries(X[ok]), equal_nan=True)
    # a forced cap, and a lone individual that only mutates
    P[6] = (0, 0, 0.3)
    X, S, n = _check_replay(P, N, seed=5, max_events=40)
    capped = n == 40
    assert capped[6] and np.all(X[6] == -1) and np.isnan(S[6]).all()
    assert np.all(X[~capped & (n > 0)] >= 0)


def test_launch_independence():
    from elfi_b200 import ops
    rs = np.random.RandomState(3)
    P = np.column_stack([rs.uniform(0.005, 2.005, 20000), np.zeros(20000), np.full(20000, 0.198)])
    X, S, n = (_np(t) for t in ops.sim_bdm(P, 20, seed=9, offset=100))
    X2, S2, n2 = (_np(t) for t in ops.sim_bdm(P, 20, seed=9, offset=100))
    assert np.array_equal(X, X2) and np.array_equal(S, S2, equal_nan=True) and np.array_equal(n, n2)
    for lo, hi in ((0, 7), (7, 12345), (12345, 20000)):
        Xs, Ss, ns = (_np(t) for t in ops.sim_bdm(P[lo:hi], 20, seed=9, offset=100 + lo))
        assert np.array_equal(Xs, X[lo:hi]) and np.array_equal(ns, n[lo:hi])
        assert np.array_equal(Ss, S[lo:hi], equal_nan=True)


@pytest.mark.parametrize('N,n_t2', [(20, 20), (20, 7), (473, 20), (473, 473), (1024, 50.5)])
def test_fused_equals_unfused_and_numpy(N, n_t2):
    import torch
    from elfi_b200 import ops
    rs = np.random.RandomState(N)
    P = np.column_stack([rs.uniform(0.5, 2.0, 3000), rs.uniform(0, 0.4, 3000), np.full(3000, 0.198)])
    X, S, _ = ops.sim_bdm(P, N, seed=2, n=n_t2)
    _, S_only, _ = ops.sim_bdm(P, N, seed=2, n=n_t2, want_data=False)
    Xh = _np(X)
    assert np.array_equal(_np(S_only), _np(S), equal_nan=True)
    assert np.array_equal(_np(ops.bdm_summaries(X, n_t2)), _np(S), equal_nan=True)
    assert np.array_equal(_host_summaries(Xh, n_t2), _np(S), equal_nan=True)
    # a strided view: column-major storage, every other row
    view = X.t().contiguous().t()[::2]
    assert view.stride() == (2, X.shape[0])
    want = _host_summaries(Xh[::2], n_t2)
    assert np.array_equal(_np(ops.bdm_summaries(view, n_t2)), want, equal_nan=True)


def _sim_law(point, B, seed):
    from elfi_b200 import ops
    X, S, n = ops.sim_bdm(np.tile(point[:3], (B, 1)), int(point[3]), seed=seed, want_data=False)
    S = _np(S)
    assert np.all(_np(n) > 0)
    return S[:, 0]


@pytest.mark.parametrize('i', range(4))
def test_law_matches_executable(i):
    g = load_golden('bdm_law')
    point = g['points'][i]
    t1_ref, clusters_ref, pop_ref = g['t1_%d' % i], g['clusters_%d' % i], g['pop_%d' % i]
    t1 = _sim_law(point, 200000, seed=100 + i)
    extinct_ref, extinct = np.isnan(t1_ref), np.isnan(t1)
    # extinction fraction within 4 standard errors
    p_ref, p = extinct_ref.mean(), extinct.mean()
    se = np.sqrt(max(p_ref * (1 - p_ref), 1e-12) / len(t1_ref) + max(p * (1 - p), 1e-12) / len(t1))
    assert abs(p - p_ref) <= 4 * se + 1e-12, (p, p_ref)
    if point[1] == 0:
        assert not extinct.any() and not extinct_ref.any()
    live_ref = ~extinct_ref
    # T1 on the surviving rows; the number of clusters is T1 * N there (pop = N)
    assert np.all(pop_ref[live_ref] == point[3])
    pv = ss.ks_2samp(t1[~extinct], t1_ref[live_ref]).pvalue
    assert pv > 1e-3, pv
    c = np.round(t1[~extinct] * point[3])
    c_ref = clusters_ref[live_ref]
    se = np.sqrt(c.var() / c.size + c_ref.var() / c_ref.size)
    assert abs(c.mean() - c_ref.mean()) <= 4 * se, (c.mean(), c_ref.mean(), se)
    print('point', point, 'KS p %.3g, extinct %.4f vs %.4f, clusters %.3f vs %.3f' % (
        pv, p, p_ref, c.mean(), c_ref.mean()))


def test_device_rejection_matches_reference_posterior():
    import elfi_b200 as elfi
    from elfi_b200.examples import bdm
    g = load_golden('bdm_rejection')
    m, dp = bdm.get_device_model()
    res = elfi.Rejection(m['d'], batch_size=100000, seed=1).sample(20000, quantile=0.1, bar=False)
    a = res.samples['alpha']
    a = a.cpu().numpy() if hasattr(a, 'cpu') else np.asarray(a)
    ref = g['alpha']
    se = np.sqrt(ref.var() / ref.size + a.var() / a.size)
    print('posterior mean %.4f vs reference %.4f (se %.4f)' % (a.mean(), ref.mean(), se))
    assert abs(a.mean() - ref.mean()) <= 4 * se
    smc = elfi.SMC(m['d'], batch_size=20000, seed=4, device_proposal=dp).sample(
        2000, quantiles=[0.5, 0.2], bar=False)
    assert len(smc.populations) == 2
    m3, _ = bdm.get_device_model(seed_obs=3)
    assert m3.observed['BDM'].sum() == 20
