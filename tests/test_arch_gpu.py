"""Device ARCH(1) simulator and summaries.

* sim_arch element by element against the NumPy replay of its Philox stream (tests/arch_replay.py),
  within a bound carried through the recurrence from the replayed normals' error; row counters
  across 2^32; split launches equal one launch;
* arch_summaries equals NumPy bit for bit on strided views and on the crafted golden rows, and the
  fused summaries equal the unfused chain bit for bit;
* statistics against the host simulator, the Rejection posterior against the host model's, and
  the samplers.
"""
from itertools import combinations

import numpy as np
import pytest
import scipy.stats as ss

import arch_replay as ar
from conftest import load_golden

pytestmark = pytest.mark.gpu
CORNERS = [(1.0, 0.0), (1.0, 1.0), (-1.0, 0.0), (-1.0, 1.0)]


def _np(t):
    return t.cpu().numpy()


def _reference_summaries(x, n_lags):
    from elfi_b200.examples import arch
    with np.errstate(all='ignore'):
        cols = [arch.sample_mean(x), arch.sample_variance(x)]
        cols += [arch.autocorr(x, i) for i in range(1, n_lags + 1)]
        cols += [arch.pairwise_autocorr(x, i, j) for i, j in combinations(range(1, n_lags + 1), 2)]
    return np.column_stack(cols)


def _same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True) and \
        np.array_equal(np.signbit(a[a == 0]), np.signbit(b[a == 0]))


# ---------------------------------------------------------------------------- sim_arch
@pytest.mark.parametrize('offset', [0, 2 ** 32 - 300])
@pytest.mark.parametrize('n_obs', [2, 3, 100, 128])
def test_sim_arch_matches_replay(offset, n_obs):
    from elfi_b200 import ops
    rs = np.random.RandomState(n_obs + offset % 89)
    B = 1000
    P = np.column_stack([rs.uniform(-1, 1, B), rs.uniform(0, 1, B)])
    P[:5] = [(0.3, 0.7)] + CORNERS
    Y, _ = ops.sim_arch(P, n_obs, n_lags=1, seed=7, offset=offset, want_data=True,
                        want_summaries=False)
    Y = _np(Y)
    want, err = ar.sim_arch(P, n_obs, seed=7, offset=offset)
    bad = ~(np.abs(Y - want) <= err)
    assert not bad.any(), (np.argwhere(bad)[:5], np.abs(Y - want)[bad][:5], err[bad][:5])
    # a wrong stream would be O(1) off: the bound is tight enough to tell
    assert np.median(err / np.maximum(np.abs(want), 1e-300)) < 1e-11


def test_sim_arch_split_launches_equal_one_launch():
    from elfi_b200 import ops
    rs = np.random.RandomState(2)
    P = np.column_stack([rs.uniform(-1, 1, 1000), rs.uniform(0, 1, 1000)])
    base = 2 ** 32 - 400
    whole = ops.sim_arch(P, 100, 5, seed=9, offset=base, want_data=True)
    for cut in (1, 400, 777):
        parts = [ops.sim_arch(P[:cut], 100, 5, seed=9, offset=base, want_data=True),
                 ops.sim_arch(P[cut:], 100, 5, seed=9, offset=base + cut, want_data=True)]
        for j in range(2):
            joined = np.concatenate([_np(parts[0][j]), _np(parts[1][j])])
            assert np.array_equal(joined, _np(whole[j]), equal_nan=True), (cut, j)


# ---------------------------------------------------------------------------- bit-for-bit summaries
@pytest.mark.parametrize('n,n_lags', [(2, 1), (7, 6), (8, 3), (17, 8), (100, 5), (101, 8), (128, 8)])
def test_summaries_equal_numpy_on_strided_views(n, n_lags):
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    rs = np.random.RandomState(n)
    B = 3000
    full = rs.randn(B, n + 1) * rs.uniform(1e-3, 1e3, (B, 1)) + rs.uniform(-5, 5, (B, 1))
    full[0] = 2.0
    full[1] = 0.0
    full[2, 1 + rs.randint(n)] = np.nan
    full[3, 1 + rs.randint(n)] = np.inf
    y = full[:, 1:]                                   # the reference's (n + 1)-strided view
    want = _reference_summaries(y, n_lags)
    d = dev.to_device(full)
    for src in (d[:, 1:], dev.to_device(y), dev.to_device(y.T.copy()).T):
        assert _same_bits(_np(ops.arch_summaries(src, n_lags)), want), src.stride()


def test_summaries_equal_golden_crafted_rows():
    from elfi_b200 import ops
    g = load_golden('arch_summaries')
    draws = load_golden('arch_draws')
    data = dict(y1=draws['y1'], yb=draws['yb'], ys=draws['ys'], crafted=g['crafted'], n2=g['n2'],
                n128=g['n128'])
    for key in (k for k in g if '_L' in k):
        name, L = key.rsplit('_L', 1)
        assert _same_bits(_np(ops.arch_summaries(data[name], int(L))), g[key]), key


@pytest.mark.parametrize('B', [1, 129, 100003])
def test_fused_summaries_equal_unfused_chain(B):
    from elfi_b200 import ops
    rs = np.random.RandomState(B % 1000)
    P = np.column_stack([rs.uniform(-1, 1, B), rs.uniform(0, 1, B)])
    P[:min(B, 5)] = ([(0.3, 0.7)] + CORNERS)[:min(B, 5)]
    for n_obs, n_lags in ((100, 5), (128, 8), (2, 1), (33, 4)):
        Y, S = ops.sim_arch(P, n_obs, n_lags, seed=3, offset=2 ** 32 - 1000, want_data=True)
        _, S_only = ops.sim_arch(P, n_obs, n_lags, seed=3, offset=2 ** 32 - 1000)
        chain = ops.arch_summaries(Y, n_lags)
        assert _same_bits(_np(S), _np(chain)), (n_obs, n_lags)
        assert _same_bits(_np(S_only), _np(S)), (n_obs, n_lags)
        if B <= 129:
            assert _same_bits(_np(S), _reference_summaries(_np(Y), n_lags)), (n_obs, n_lags)


# ---------------------------------------------------------------------------- statistics
@pytest.mark.parametrize('params', [(0.3, 0.7)] + CORNERS)
def test_statistics_match_host_simulator(params):
    from elfi_b200 import ops
    from elfi_b200.examples import arch
    B = 20000
    with np.errstate(all='ignore'):
        y_h = arch.arch(*params, batch_size=B, random_state=np.random.RandomState(1))
    host = _reference_summaries(y_h, 5)
    _, S = ops.sim_arch(np.tile(params, (B, 1)), 100, 5, seed=77)
    S = _np(S)
    for j, name in ((0, 'MU'), (1, 'VAR'), (2, 'AC_1'), (3, 'AC_2'), (7, 'PW_1_2')):
        p = ss.ks_2samp(S[:, j], host[:, j]).pvalue
        assert p > 1e-5, (params, name, p)


def test_device_rejection_posterior_matches_host():
    import elfi_b200 as elfi
    from elfi_b200.examples import arch
    host_m = arch.get_model(seed_obs=2)
    res_h = elfi.Rejection(host_m['d'], batch_size=10000, seed=1).sample(300, quantile=0.01,
                                                                          bar=False)
    m, dp = arch.get_device_model(seed_obs=2)
    assert np.array_equal(m.observed['Y'], host_m.observed['Y'])
    res_d = elfi.Rejection(m['d'], batch_size=100000, seed=1).sample(3000, quantile=0.01, bar=False)
    for name in ('t1', 't2'):
        h, d = res_h.samples[name], res_d.samples[name]
        se = np.sqrt(h.var() / len(h) + d.var() / len(d))
        assert abs(h.mean() - d.mean()) < 4 * se, (name, h.mean(), d.mean(), se)


# ---------------------------------------------------------------------------- samplers
def test_device_model_smc_and_adaptive_distance_smc():
    import elfi_b200 as elfi
    from elfi_b200.examples import arch
    m, dp = arch.get_device_model(seed_obs=3)

    def run(**kw):
        return elfi.SMC(m['d'], batch_size=10000, seed=4, device_proposal=dp, **kw).sample(
            1000, quantiles=[0.1, 0.3, 0.3], bar=False)
    smc = run()
    assert len(smc.populations) == 3 and np.all(np.isfinite(smc.weights))
    assert abs(smc.sample_means['t1'] - 0.3) < 0.3
    par = run(distributed=False, max_parallel_batches=2)
    par2 = run(distributed=False, max_parallel_batches=2)
    assert np.array_equal(par.samples_array, par2.samples_array)
    assert np.array_equal(par.weights, par2.weights)

    names = ['MU', 'VAR'] + ['AC_{}'.format(i) for i in range(1, 6)] + \
        ['PW_{}_{}'.format(i, j) for i, j in combinations(range(1, 6), 2)]
    m['d'].become(elfi.AdaptiveDistance(*[m[n] for n in names]))
    ad = elfi.AdaptiveDistanceSMC(m['d'], batch_size=10000, seed=5, device_proposal=dp).sample(
        1000, rounds=3, quantile=0.3, bar=False)
    assert len(ad.populations) == 3
    assert np.all(np.isfinite(ad.samples_array))
