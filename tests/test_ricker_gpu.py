"""Device Poisson sampler, Ricker simulators, summaries and chi_squared.

* ops.poisson equals the NumPy replay (tests/ricker_replay.py) element by element, apart from a
  counted handful of knife-edge decisions, fits scipy.stats.poisson, and gives NaN where NumPy
  raises;
* sim_ricker, one step at a time (the map is chaotic, so whole rows cannot be compared): N_t is
  the replayed update of the kernel's own N_{t-1}, Y_t the replayed Poisson draw at phi N_t;
  row counters across 2^32, split launches, the deterministic model;
* the fused summaries, ricker_summaries and chi_squared equal NumPy bit for bit;
* statistics against the host stochastic_ricker, Rejection posteriors, and the samplers.
"""
import numpy as np
import pytest
import scipy.stats as ss

import ricker_replay as rr

pytestmark = pytest.mark.gpu
EPS = 2.0 ** -52


def _np(t):
    return t.cpu().numpy()


# ---------------------------------------------------------------------------- ops.poisson
def test_poisson_matches_replay():
    from elfi_b200 import ops
    rs = np.random.RandomState(0)
    lam = np.concatenate([rs.uniform(0, 10, 20000), 10 ** rs.uniform(1, 18.9, 20000),
                          [0.0, 1e-300, 10.0, np.nextafter(10.0, 0), rr.LAM_MAX]])
    for offset in (0, 2 ** 32 - 7000):
        got = _np(ops.poisson(lam, seed=11, offset=offset))
        k, trials, margin, kind = rr.poisson_ops(lam, 11, offset)
        amb = rr.ambiguous(margin, kind)
        assert amb.sum() <= 5, amb.sum()
        assert np.array_equal(got[~amb], k[~amb]), np.flatnonzero((got != k) & ~amb)[:10]
        assert trials.max() <= rr.MAX_TRIALS - 20


@pytest.mark.parametrize('lam', [0.0, 1e-3, 0.5, 5.0, np.nextafter(10.0, 0), 10.0, 37.0, 1e3, 1e6,
                                 1e12, 1e15])
def test_poisson_goodness_of_fit(lam):
    from elfi_b200 import ops
    n = 10 ** 6
    k = _np(ops.poisson(np.full(n, lam), seed=int(lam * 1000) % 2 ** 31 + 1))
    assert np.all(k == np.floor(k)) and np.all(k >= 0)
    if lam == 0.0:
        assert np.all(k == 0)
        return
    dist = ss.poisson(lam)
    if lam < 1e9:
        # bins of at least ~50 expected counts from the quantiles of the exact distribution
        edges = np.unique(dist.ppf(np.linspace(0, 1, 201)[1:-1]))
        idx = np.searchsorted(edges, k, side='left')
        obs = np.bincount(idx, minlength=len(edges) + 1)
        cdf = np.concatenate([[0.0], dist.cdf(edges), [1.0]])
        # bin b holds edges[b-1] < k <= edges[b]
        exp = np.diff(cdf) * n
        keep = exp > 0
        chi2 = np.sum((obs[keep] - exp[keep]) ** 2 / exp[keep])
        p = ss.chi2.sf(chi2, keep.sum() - 1)
    else:
        # beyond double's integer resolution of a bin test: the standardised counts are normal
        p = ss.kstest((k - lam) / np.sqrt(lam), 'norm').pvalue
        assert abs(k.mean() - lam) < 5 * np.sqrt(lam / n)
    assert p > 1e-4, (lam, p)


def test_poisson_nan_where_numpy_raises():
    from elfi_b200 import ops
    lam = np.array([-1.0, -1e-300, np.nan, np.inf, np.nextafter(rr.LAM_MAX, np.inf), 1e30])
    assert np.isnan(_np(ops.poisson(lam, seed=1))).all()


# ---------------------------------------------------------------------------- sim_ricker
def _one_step_checks(P, n_obs, seed, offset, stock_init=1.0):
    """N_t and Y_t of sim_ricker against the replayed step from the kernel's own N_{t-1}."""
    from elfi_b200 import ops
    Y, N, S = ops.sim_ricker(P, n_obs, seed=seed, offset=offset, stock_init=stock_init,
                             want_data=True, want_latent=True, want_summaries=False)
    Y, N = _np(Y), _np(N)
    B = P.shape[0]
    r, sigma, phi = P[:, 0:1], P[:, 1:2], P[:, 2:3]
    e, rad = rr.ricker_normals(B, n_obs, seed, offset)
    prev = np.concatenate([np.full((B, 1), float(stock_init)), N[:, :-1]], axis=1)
    with np.errstate(all='ignore'):
        arg = (r - prev) + sigma * e
        want = prev * np.exp(arg)
        # e is within 1e-14 max(1, rad) of the device's; exp and the roundings add a few ulp
        rel = np.abs(sigma) * 1e-14 * np.maximum(1.0, rad) + 2 * EPS * np.abs(arg) + 8 * EPS
        ok = (np.abs(N - want) <= rel * np.abs(want) + 1e-300) | ((N == want) & np.isfinite(want))
    assert ok.all(), np.argwhere(~ok)[:5]
    k, trials, margin, kind = rr.ricker_counts(phi * N, B, n_obs, seed, offset)
    amb = rr.ambiguous(margin, kind)
    assert amb.sum() <= max(5, amb.size // 100000), amb.sum()
    assert np.array_equal(Y[~amb], k[~amb], equal_nan=True)
    return Y, N


@pytest.mark.parametrize('offset', [0, 2 ** 32 - 300])
def test_sim_ricker_one_step_replay(offset):
    rs = np.random.RandomState(offset % 97)
    B = 600
    # prior-predictive rows (extinction, rates up to ~1e10 and beyond) and the default truth
    P = np.column_stack([np.e + rs.exponential(2.0, B), ss.truncnorm.rvs(0, 5, size=B, random_state=rs),
                         rs.uniform(0, 100, B)])
    P[:50] = [3.8, 0.3, 10.0]
    Y, N = _one_step_checks(P, 50, seed=5, offset=offset)
    assert (N[:, -1] == 0).any() and (Y == 0).any() and np.nanmax(Y) > 1e6


def test_sim_ricker_split_launches_equal_one_launch():
    from elfi_b200 import ops
    rs = np.random.RandomState(2)
    P = np.column_stack([rs.uniform(1, 6, 1000), rs.uniform(0, 1, 1000), rs.uniform(1, 50, 1000)])
    base = 2 ** 32 - 400
    whole = ops.sim_ricker(P, 30, seed=9, offset=base, want_data=True, want_latent=True,
                           want_summaries=True)
    for cut in (1, 400, 777):
        parts = [ops.sim_ricker(P[:cut], 30, seed=9, offset=base, want_data=True, want_latent=True,
                                want_summaries=True),
                 ops.sim_ricker(P[cut:], 30, seed=9, offset=base + cut, want_data=True,
                                want_latent=True, want_summaries=True)]
        for j in range(3):
            joined = np.concatenate([_np(parts[0][j]), _np(parts[1][j])])
            assert np.array_equal(joined, _np(whole[j]), equal_nan=True), (cut, j)


def test_sim_ricker_deterministic():
    from elfi_b200 import ops
    from elfi_b200.examples import ricker
    r = np.array([0.5, 2.0, 3.8, 6.0, 12.0, np.nan])
    for stock_init in (1.0, 0.25):
        Y, N, S = ops.sim_ricker(r, 40, stochastic=False, stock_init=stock_init, want_data=True,
                                 want_latent=True)
        Y, N = _np(Y), _np(N)
        assert np.array_equal(Y, N, equal_nan=True) and np.all(Y[:, 0] == stock_init)
        prev = Y[:, :-1]
        with np.errstate(all='ignore'):
            want = prev * np.exp(r[:, None] - prev)
            ok = (np.abs(Y[:, 1:] - want) <= 8 * EPS * np.abs(want)) | (np.isnan(want) & np.isnan(Y[:, 1:]))
        assert ok.all()
        host = ricker.ricker(r[:3], stock_init=stock_init, n_obs=5, batch_size=3)
        assert np.allclose(Y[:3, :5], host, rtol=1e-13)        # before chaos takes over


# ---------------------------------------------------------------------------- bit-for-bit summaries
@pytest.mark.parametrize('n_obs', [1, 7, 8, 50, 128, 129, 300])
def test_fused_summaries_equal_ricker_summaries_and_numpy(n_obs):
    from elfi_b200 import ops
    from elfi_b200.examples import ricker
    rs = np.random.RandomState(n_obs)
    P = np.column_stack([np.e + rs.exponential(2.0, 3000), rs.uniform(0, 2, 3000),
                         rs.uniform(0, 100, 3000)])
    Y, _, S = ops.sim_ricker(P, n_obs, seed=3, offset=2 ** 32 - 1000, want_data=True)
    S2 = ops.ricker_summaries(Y)
    assert np.array_equal(_np(S), _np(S2), equal_nan=True)
    y = _np(Y)
    with np.errstate(invalid='ignore'):
        want = np.column_stack([ricker.ss_mean(y), ricker.ss_var(y), ricker.num_zeros(y)])
    assert np.array_equal(_np(S), want, equal_nan=True)


def test_ricker_summaries_and_chi_squared_equal_numpy_on_device_data():
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    from elfi_b200.examples import ricker
    rs = np.random.RandomState(4)
    y = rs.poisson(rs.choice([0.0, 0.3, 4.0, 1e3, 1e9], size=(4000, 1)), size=(4000, 50)).astype(float)
    y[5, 7] = np.nan
    view = dev.to_device(np.concatenate([y, rs.randn(4000, 3)], axis=1))[:, :50]
    host = [ricker.ss_mean(y), ricker.ss_var(y), ricker.num_zeros(y)]
    for src in (dev.to_device(y), view):
        S = ops.ricker_summaries(src)
        assert np.array_equal(_np(S), np.column_stack(host), equal_nan=True)
        devs = [ricker.ss_mean(src), ricker.ss_var(src), ricker.num_zeros(src)]
        for row in (0, int(np.argmin(host[2])), int(np.argmax(host[2]))):
            obs = tuple(v[row:row + 1] for v in host)
            with np.errstate(divide='ignore', invalid='ignore'):
                want = ricker.chi_squared(*host, observed=obs)
            got = _np(ricker.chi_squared(*devs, observed=obs))
            assert np.array_equal(got, want, equal_nan=True), row
        zero_obs = (np.zeros(1), np.zeros(1), np.array([50]))
        with np.errstate(divide='ignore', invalid='ignore'):
            want = ricker.chi_squared(*host, observed=zero_obs)
        assert np.array_equal(_np(ricker.chi_squared(*devs, observed=zero_obs)), want, equal_nan=True)
        assert np.isnan(want).any() and np.isinf(want).any()
    K = 128
    Sk = rs.randn(300, K) ** 2
    ok = rs.randn(K) ** 2
    ok[3] = 0.0
    with np.errstate(divide='ignore', invalid='ignore'):
        want = ricker.chi_squared(*Sk.T, observed=tuple(ok[:, None]))
    assert np.array_equal(_np(ops.chi_squared(Sk, ok)), want, equal_nan=True)


# ---------------------------------------------------------------------------- statistics
def _host_ricker_with_stock(params, n_obs, B, seed):
    """stochastic_ricker's loop (ricker.py:73-85) that also returns the last latent stock."""
    rs = np.random.RandomState(seed)
    r, std, scale = params
    y = np.empty((B, n_obs))
    prev = 1.0
    for ii in range(n_obs):
        stock = prev * np.exp(r - prev + std * rs.randn(B))
        prev = stock
        y[:, ii] = rs.poisson(scale * stock, B)
    return y, stock


@pytest.mark.parametrize('params', [(3.8, 0.3, 10.0), (2.0, 0.1, 50.0), (6.0, 1.0, 1.0)])
def test_statistics_match_host_simulator(params):
    from elfi_b200 import ops
    from elfi_b200.examples import ricker
    B = 20000
    y_h, stock_h = _host_ricker_with_stock(params, 50, B, seed=1)
    assert np.nanmax(params[2] * stock_h) < 1e10
    _, N, S = ops.sim_ricker(np.tile(params, (B, 1)), 50, seed=77, want_latent=True)
    S = _np(S)
    host = [ricker.ss_mean(y_h), ricker.ss_var(y_h), ricker.num_zeros(y_h)]
    for j in range(2):
        assert ss.ks_2samp(S[:, j], host[j]).pvalue > 1e-3, (params, j)
    zd, zh = S[:, 2].astype(np.int64), host[2].astype(np.int64)
    counts = np.array([np.bincount(zd, minlength=51), np.bincount(zh, minlength=51)])
    counts = counts[:, counts.sum(axis=0) >= 20]
    if counts.shape[1] > 1:
        assert ss.chi2_contingency(counts)[1] > 1e-3, params
    ext_d, ext_h = np.mean(_np(N)[:, -1] == 0), np.mean(stock_h == 0)
    se = np.sqrt(max(ext_h * (1 - ext_h), 1.0 / B) / B * 2)
    assert abs(ext_d - ext_h) < 5 * se, (ext_d, ext_h)


def test_device_rejection_posterior_matches_host():
    import elfi_b200 as elfi
    from elfi_b200.examples import ricker
    host_m = ricker.get_model(seed_obs=2)
    res_h = elfi.Rejection(host_m['d'], batch_size=5000, seed=1).sample(300, quantile=0.01,
                                                                         bar=False)
    m, dp = ricker.get_device_model(seed_obs=2)
    assert np.array_equal(m.observed['Ricker'], host_m.observed['Ricker'])
    res_d = elfi.Rejection(m['d'], batch_size=100000, seed=1).sample(3000, quantile=0.01, bar=False)
    for name in ('t1', 't2', 't3'):
        h, d = res_h.samples[name], res_d.samples[name]
        se = np.sqrt(h.var() / len(h) + d.var() / len(d))
        assert abs(h.mean() - d.mean()) < 4 * se, (name, h.mean(), d.mean(), se)


# ---------------------------------------------------------------------------- samplers
@pytest.mark.parametrize('stochastic', [True, False])
def test_device_models_rejection_and_smc(stochastic):
    import elfi_b200 as elfi
    from elfi_b200.examples import ricker
    m, dp = ricker.get_device_model(seed_obs=3, stochastic=stochastic)
    res = elfi.Rejection(m['d'], batch_size=20000, seed=1).sample(200, quantile=0.01, bar=False)
    assert res.n_samples == 200 and not np.any(np.isnan(res.discrepancies))
    if stochastic:
        assert abs(res.sample_means['t1'] - 3.8) < 1.5

    def run(**kw):
        return elfi.SMC(m['d'], batch_size=10000, seed=4, device_proposal=dp, **kw).sample(
            1000, quantiles=[0.1, 0.3, 0.3], bar=False)
    smc = run()
    assert len(smc.populations) == 3 and np.all(np.isfinite(smc.weights))
    par = run(distributed=False, max_parallel_batches=2)
    par2 = run(distributed=False, max_parallel_batches=2)
    assert np.array_equal(par.samples_array, par2.samples_array)
    assert np.array_equal(par.weights, par2.weights)
