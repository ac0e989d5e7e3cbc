"""Device g-and-k robust / octile summaries, the fused simulators, sim_bignk and euclidean_multiss.

* gnk_summaries equals the reference's NumPy ss_robust / ss_octile bit for bit (series lengths
  around the warp and register-network boundaries, d = 1 and 2, strided views, NaN / inf / ties);
* the fused simulators equal their unfused chain (simulator, then gnk_summaries) bit for bit, for
  row counters that straddle 2^32 and for offset slices;
* sim_bignk's data equals a NumPy replay of its Philox stream (oracle/streams.py) element by
  element at the ulp tolerances of tests/test_streams_gpu.py;
* statistics against the host BiGNK, euclidean_multiss bit for bit, and the samplers.
"""
import numpy as np
import pytest
import scipy.stats as ss

import streams

pytestmark = pytest.mark.gpu

KINDS = ('ss_robust', 'ss_octile')
SALT_SIM_BIGNK = 0x42474E4B


def _np(t):
    return t.cpu().numpy()


def _host(y, kind):
    from elfi_b200.examples import gnk
    with np.errstate(invalid='ignore'):
        return (gnk.ss_robust if kind == 'ss_robust' else gnk.ss_octile)(y)[:, :, 0]


def _edge_rows(n, d, rs):
    rows = [rs.randn(n, d), np.round(rs.randn(n, d)), np.full((n, d), 0.75), rs.randn(n, d),
            rs.randn(n, d), rs.randn(n, d)]
    rows[3][rs.rand(n) < 0.3] = np.inf
    rows[4][rs.rand(n) < 0.3] = -np.inf
    rows[5][rs.randint(n), rs.randint(d)] = np.nan
    return np.stack(rows)


@pytest.mark.parametrize('d', [1, 2])
@pytest.mark.parametrize('n', [1, 2, 3, 7, 8, 31, 32, 33, 50, 150, 256, 511, 512, 513, 1000, 2048])
def test_gnk_summaries_match_numpy(n, d):
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    rs = np.random.RandomState(n * 10 + d)
    y = np.concatenate([rs.standard_t(3, size=(300, n, d)), _edge_rows(n, d, rs)])
    # unaligned view: a row pitch of n + 3 observations and an odd element offset
    buf = dev.to_device(rs.randn(len(y) * (n + 3) * d + 1))
    view = buf[1:].reshape(len(y), n + 3, d)[:, 1:n + 1, :]
    view.copy_(dev.to_device(y))
    for kind in KINDS:
        want = _host(y, kind)
        for src in (dev.to_device(y), view):
            got = _np(ops.gnk_summaries(src, kind))
            assert np.array_equal(got, want, equal_nan=True), (kind, n, d)


def _rows(B, rs):
    return [rs.uniform(0, 10, B), rs.uniform(0.1, 10, B), rs.uniform(0, 10, B), rs.uniform(0, 10, B)]


N_OBS = [1, 2, 3, 50, 63, 64, 150, 256, 512]


@pytest.mark.parametrize('n_obs', N_OBS)
def test_fused_univariate_equals_unfused(n_obs):
    from elfi_b200 import ops
    rs = np.random.RandomState(n_obs)
    B = 3000
    cols = _rows(B, rs)
    for seed, offset in ((7, 0), (2 ** 32 + 9, 2 ** 32 - 1500)):
        Y = ops.sim_gnk(*cols, n_obs=n_obs, seed=seed, offset=offset)
        for kind in KINDS:
            want = _np(ops.gnk_summaries(Y, kind))
            got = _np(ops.sim_gnk_summaries(*cols, n_obs=n_obs, seed=seed, offset=offset, kind=kind))
            assert np.array_equal(got, want, equal_nan=True), (n_obs, seed, offset, kind)
            part = _np(ops.sim_gnk_summaries(*[c[1000:2100] for c in cols], n_obs=n_obs, seed=seed,
                                             offset=offset + 1000, kind=kind))
            assert np.array_equal(part, want[1000:2100], equal_nan=True)


def _bignk_params(B, rs):
    P = np.column_stack([rs.uniform(0, 5, B), rs.uniform(0, 5, B), rs.uniform(0.01, 5, B),
                         rs.uniform(0.01, 5, B), rs.uniform(-5, 5, B), rs.uniform(-5, 5, B),
                         rs.uniform(-.5, 5, B), rs.uniform(-.5, 5, B), rs.uniform(-1, 1, B)])
    edges = [1.0, -1.0, 0.0, 1.0 + 1e-12][:B]     # both edges, independence, just outside
    P[:len(edges), 8] = edges
    return P


@pytest.mark.parametrize('n_obs', N_OBS)
def test_fused_bivariate_equals_unfused(n_obs):
    from elfi_b200 import ops
    rs = np.random.RandomState(100 + n_obs)
    P = _bignk_params(3000, rs)
    for seed, offset in ((7, 0), (2 ** 32 + 9, 2 ** 32 - 1500)):
        Y, _ = ops.sim_bignk(P, n_obs=n_obs, seed=seed, offset=offset)
        y = _np(Y)
        assert np.isnan(y[3]).all() and not np.isnan(y[:3]).any()
        for kind in KINDS:
            want = _np(ops.gnk_summaries(Y, kind))
            Y2, got = ops.sim_bignk(P, n_obs=n_obs, seed=seed, offset=offset, kind=kind)
            assert np.array_equal(_np(got), want, equal_nan=True), (n_obs, seed, offset, kind)
            assert np.array_equal(_np(Y2), y, equal_nan=True)
            _, part = ops.sim_bignk(P[1000:2100], n_obs=n_obs, seed=seed, offset=offset + 1000,
                                    want_data=False, kind=kind)
            assert np.array_equal(_np(part), want[1000:2100], equal_nan=True)


def replay_bignk(P, c, n_obs, seed, offset):
    """sim_bignk_kernel in NumPy: block (row, j) -> n0, n1; z1 = n0 (NaN when |rho| > 1),
    z2 = rho n0 + sqrt(1 - rho^2) n1; y = gnk_quantile.  Returns (Y (B, n_obs, 2), error bound)."""
    B = len(P)
    j = np.arange(n_obs, dtype=np.uint64)[None, :]
    n0, n1, rad = streams.normal2(streams._block(streams.rows_of(B, offset)[:, None], j,
                                                 SALT_SIM_BIGNK, seed))
    rho = P[:, 8:9]
    with np.errstate(invalid='ignore'):
        sr = np.sqrt(1.0 - rho * rho)
        z = np.stack([np.where(np.abs(rho) <= 1.0, n0, np.nan), rho * n0 + sr * n1], axis=2)
        A, Bs, g, k = (P[:, [a, a + 1]][:, None, :] for a in (0, 2, 4, 6))
        Y = streams.gnk_quantile(A, Bs, g, k, c, z)
        kurt = (1.0 + z * z) ** k
        slope = np.abs(Bs) * (1.0 + abs(c)) * kurt * (1.0 + 2.0 * np.abs(k) + np.abs(g * z))
        zerr = 1e-14 * np.maximum(1.0, rad)[:, :, None] * 2.0 + 4e-16 * np.abs(z)
        err = 1e-12 * (np.abs(A) + np.abs(Y - A)) + slope * zerr
    return Y, err


@pytest.mark.parametrize('B,n_obs,seed,offset', [(1, 1, 3, 0), (257, 150, 3, 7),
                                                 (1000, 33, 2 ** 32 + 5, 2 ** 32 - 500)])
def test_sim_bignk_matches_replay(B, n_obs, seed, offset):
    from elfi_b200 import ops
    P = _bignk_params(B, np.random.RandomState(B))
    Y = _np(ops.sim_bignk(P, n_obs=n_obs, seed=seed, offset=offset)[0])
    Yr, err = replay_bignk(P, 0.8, n_obs, seed, offset)
    assert np.array_equal(np.isnan(Y), np.isnan(Yr))
    fin = np.isfinite(Yr)
    bad = ~(np.abs(Y[fin] - Yr[fin]) <= err[fin])
    assert not bad.any(), (int(bad.sum()), Y[fin][bad][:3], Yr[fin][bad][:3])


def test_robust_summaries_distribution_vs_host_bignk():
    """KS test of each device ss_robust column against the host BiGNK + ss_robust, 2e4 rows each."""
    from elfi_b200 import ops
    from elfi_b200.examples import bignk, gnk
    prm = [3, 4, 1, 0.5, 1, 2, .5, .4, 0.6]
    B, n_obs = 20000, 150
    y = bignk.BiGNK(*[np.full(B, v) for v in prm], n_obs=n_obs, batch_size=B,
                    random_state=np.random.RandomState(1))
    host = gnk.ss_robust(y)[:, :, 0]
    _, dev_s = ops.sim_bignk(np.tile(prm, (B, 1)), n_obs=n_obs, seed=77, want_data=False,
                             kind='ss_robust')
    dev_s = _np(dev_s)
    for col in range(8):
        p = ss.ks_2samp(dev_s[:, col], host[:, col]).pvalue
        assert p > 1e-3, (col, p)


@pytest.mark.parametrize('K', [4, 7, 8, 14])
def test_euclidean_multiss_matches_host(K):
    from elfi_b200 import device as dev
    from elfi_b200.examples import gnk
    rs = np.random.RandomState(K)
    S = rs.randn(5000, K, 1) * np.exp(rs.randn(5000, K, 1) * 3)
    obs = rs.randn(1, K, 1)
    want = gnk.euclidean_multiss(S, observed=[obs])
    got = gnk.euclidean_multiss(dev.to_device(S), observed=[obs])
    assert np.array_equal(_np(got), want)
    wide = dev.to_device(np.concatenate([S[:, :, 0], rs.randn(5000, 3)], axis=1))
    got2 = gnk.euclidean_multiss(wide[:, :K, None], observed=[obs])
    assert np.array_equal(_np(got2), want)


def test_device_models_rejection_and_smc():
    import elfi_b200 as elfi
    from elfi_b200.examples import bignk, gnk
    m, dp = bignk.get_device_model(seed=3)
    res = elfi.Rejection(m['d'], batch_size=20000, seed=1).sample(200, quantile=0.01, bar=False)
    assert res.n_samples == 200 and np.all(np.isfinite(res.discrepancies))
    assert abs(res.sample_means['a1'] - 3) < 1.5 and abs(res.sample_means['a2'] - 4) < 1.5

    def run(**kw):
        return elfi.SMC(m['d'], batch_size=10000, seed=4, device_proposal=dp, **kw).sample(
            1000, quantiles=[0.1, 0.3, 0.3], bar=False)
    smc = run()
    assert len(smc.populations) == 3 and np.all(np.isfinite(smc.weights))
    par = run(distributed=False, max_parallel_batches=2)
    par2 = run(distributed=False, max_parallel_batches=2)
    assert np.array_equal(par.samples_array, par2.samples_array)
    assert np.array_equal(par.weights, par2.weights)
    mg, prop = gnk.get_device_model(n_obs=200, seed=3, summary='ss_robust')
    res = elfi.Rejection(mg['d'], batch_size=20000, seed=1).sample(200, quantile=0.01, bar=False)
    assert res.n_samples == 200 and abs(res.sample_means['A'] - 3) < 1.0
    smc = elfi.SMC(mg['d'], batch_size=10000, seed=4, device_proposal=prop).sample(
        1000, quantiles=[0.1, 0.3], bar=False)
    assert len(smc.populations) == 2 and np.all(np.isfinite(smc.weights))
