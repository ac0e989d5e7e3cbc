"""Device M/G/1 simulator and row quantiles.

* sim_mg1 element by element against the NumPy replay of its Philox stream (tests/mg1_replay.py):
  the service times exact, the series within a bound carried through the recurrence; row counters
  across 2^32; split launches equal one launch; the rows where NumPy raises are NaN;
* row_quantiles equals np.quantile bit for bit on strided views, with NaN and inf rows and random
  levels, and on the golden rows; the fused quantiles equal the unfused chain bit for bit;
* statistics against the host simulator, the Rejection posterior against the host model's, and
  the samplers with the conditional device prior.
"""
import numpy as np
import pytest
import scipy.stats as ss

import mg1_replay as mr
from conftest import load_golden

pytestmark = pytest.mark.gpu
Q10 = np.linspace(0, 1, 10)
TRUTH = (1., 5., 0.2)
CORNERS = [(1., 5., 1e-3), (1., 5., 0.5), (3., 3., 0.2), (3., 13., 0.2)]


def _np(t):
    return t.cpu().numpy()


def _same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True) and \
        np.array_equal(np.signbit(a[a == 0]), np.signbit(b[a == 0]))


def _params(B, rs):
    t1 = rs.uniform(0, 10, B)
    P = np.column_stack([t1, t1 + rs.uniform(0, 10, B), rs.uniform(0, 0.5, B)])
    P[:5] = [TRUTH] + CORNERS
    return P


# ---------------------------------------------------------------------------- sim_mg1
@pytest.mark.parametrize('offset', [0, 2 ** 32 - 300])
@pytest.mark.parametrize('n_obs', [2, 7, 50, 512])
def test_sim_mg1_matches_replay(offset, n_obs):
    from elfi_b200 import ops
    rs = np.random.RandomState(n_obs + offset % 89)
    B = 1000
    P = _params(B, rs)
    Y, _ = ops.sim_mg1(P, n_obs, seed=7, offset=offset, want_data=True, want_summaries=False)
    Y = _np(Y)
    want, err, W, U = mr.sim_mg1(P, n_obs, seed=7, offset=offset)
    bad = ~(np.abs(Y - want) <= err)
    assert not bad.any(), (np.argwhere(bad)[:5], np.abs(Y - want)[bad][:5], err[bad][:5])
    # a wrong stream would be O(1) off: the bound is tight enough to tell
    assert np.median(err / np.abs(want)) < 1e-9
    # the first customer: y_0 = U_0 + max(0, W_0), U exact and W within the ulps of log
    first = Y[:, 0] - np.maximum(0, W[:, 0])
    assert np.all(np.abs(first - U[:, 0]) <= 4 * mr.EPS * (np.abs(Y[:, 0]) + np.abs(W[:, 0])))


def test_service_times_are_exact():
    """With t3 = inf every arrival gap is 0, so the first inter-departure time is the first service
    time plus 0: the replay's U, exactly."""
    from elfi_b200 import ops
    rs = np.random.RandomState(1)
    B, n = 500, 20
    t1 = rs.uniform(0, 10, B)
    P = np.column_stack([t1, t1 + rs.uniform(0, 10, B), np.full(B, np.inf)])
    Y, _ = ops.sim_mg1(P, n, seed=3, offset=2 ** 32 - 5, want_data=True, want_summaries=False)
    _, _, W, U = mr.sim_mg1(P, n, seed=3, offset=2 ** 32 - 5)
    assert np.all(W == 0)
    assert np.array_equal(_np(Y)[:, 0], U[:, 0])


def test_sim_mg1_split_launches_equal_one_launch():
    from elfi_b200 import ops
    P = _params(1000, np.random.RandomState(2))
    base = 2 ** 32 - 400
    whole = ops.sim_mg1(P, 50, seed=9, offset=base, want_data=True)
    for cut in (1, 400, 777):
        parts = [ops.sim_mg1(P[:cut], 50, seed=9, offset=base, want_data=True),
                 ops.sim_mg1(P[cut:], 50, seed=9, offset=base + cut, want_data=True)]
        for j in range(2):
            joined = np.concatenate([_np(parts[0][j]), _np(parts[1][j])])
            assert np.array_equal(joined, _np(whole[j]), equal_nan=True), (cut, j)


def test_rows_where_numpy_raises_are_nan():
    from elfi_b200 import ops
    P = np.array([(1, 5, -0.2), (1, 5, -0.0), (1, 5, -np.inf), (1, np.inf, 0.2), (np.nan, 5, 0.2),
                  (-np.inf, 5, 0.2), TRUTH, (1, 5, 0.0), (1, 5, np.nan), (1, 5, np.inf)])
    Y, S = ops.sim_mg1(P, 20, seed=1, want_data=True)
    Y, S = _np(Y), _np(S)
    assert np.isnan(Y[:6]).all() and np.isnan(S[:6]).all()
    assert np.isfinite(Y[6]).all() and np.isfinite(S[6]).all()
    # t3 = 0: infinite gaps, so inf then inf - inf = NaN, as NumPy computes
    assert np.isposinf(Y[7, 0]) and np.isnan(Y[7, 1:]).all()
    assert np.isnan(Y[8]).all() and np.isnan(S[8]).all()
    assert np.isfinite(Y[9]).all()


# ---------------------------------------------------------------------------- bit-for-bit quantiles
@pytest.mark.parametrize('n', [2, 3, 50, 64, 65, 512])
def test_row_quantiles_equal_numpy_on_strided_views(n):
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    rs = np.random.RandomState(n)
    B = 3000
    full = rs.exponential(1.0, (B, n + 1)) * rs.uniform(1e-3, 1e3, (B, 1))
    full[0] = 2.0
    full[1, 1:] = np.round(full[1, 1:])
    full[2, 1 + rs.randint(n)] = np.nan
    full[3, 1 + rs.randint(n)] = np.inf
    full[4, 1 + rs.randint(n)] = -np.inf
    full[5, 1:3] = [np.inf, -np.inf]
    y = full[:, 1:]
    d = dev.to_device(full)
    for q in (Q10, np.sort(rs.uniform(0, 1, 7)), rs.uniform(0, 1, 32), [1.0], [0.0, 0.5]):
        want = np.quantile(y, q, axis=1).T
        for src in (d[:, 1:], dev.to_device(y), dev.to_device(y.T.copy()).T):
            assert _same_bits(_np(ops.row_quantiles(src, q)), want), (src.stride(), len(q))


def test_row_quantiles_equal_golden_rows():
    from elfi_b200 import ops
    g = load_golden('mg1_summaries')
    d = load_golden('mg1_draws')
    for name in ('y1', 'yb', 'ys'):
        if d[name].shape[1] >= 2:
            assert _same_bits(_np(ops.row_quantiles(d[name], Q10)), g[name + '_q10']), name
    for name in ('crafted', 'n2'):
        for key, q in (('_q10', Q10), ('_qr', g['qr'])):
            got, want = _np(ops.row_quantiles(g[name], q)), g[name + key]
            # np.quantile's partition does not order -0.0 and 0.0: crafted row 7 mixes both
            assert np.array_equal(got, want, equal_nan=True), name + key
            rows = [i for i in range(len(want)) if not (name == 'crafted' and i == 7)]
            assert _same_bits(got[rows], want[rows]), name + key


@pytest.mark.parametrize('B', [1, 129, 100003])
def test_fused_quantiles_equal_unfused_chain(B):
    from elfi_b200 import ops
    rs = np.random.RandomState(B % 1000)
    P = _params(max(B, 5), rs)[:B]
    P[B // 2:B // 2 + 1] = (1, 5, -0.0)
    for n_obs, q in ((50, Q10), (512, Q10), (2, [0.5]), (33, rs.uniform(0, 1, 32))):
        Y, S = ops.sim_mg1(P, n_obs, q, seed=3, offset=2 ** 32 - 1000, want_data=True)
        _, S_only = ops.sim_mg1(P, n_obs, q, seed=3, offset=2 ** 32 - 1000)
        chain = ops.row_quantiles(Y, q)
        assert _same_bits(_np(S), _np(chain)), n_obs
        assert _same_bits(_np(S_only), _np(S)), n_obs
        if B <= 129:
            assert _same_bits(_np(S), np.quantile(_np(Y), q, axis=1).T), n_obs


# ---------------------------------------------------------------------------- statistics
@pytest.mark.parametrize('params', [TRUTH] + CORNERS)
def test_statistics_match_host_simulator(params):
    from elfi_b200 import ops
    from elfi_b200.examples import mg1
    B = 20000
    y_h = mg1.MG1(*params, batch_size=B, random_state=np.random.RandomState(1))
    host = np.quantile(y_h, Q10, axis=1).T
    _, S = ops.sim_mg1(np.tile(params, (B, 1)), 50, Q10, seed=77)
    S = _np(S)
    for j in (0, 2, 5, 9):
        p = ss.ks_2samp(S[:, j], host[:, j]).pvalue
        assert p > 1e-5, (params, j, p)


def test_device_rejection_posterior_matches_host():
    import elfi_b200 as elfi
    from elfi_b200.examples import mg1
    host_m = mg1.get_model(seed_obs=2)
    res_h = elfi.Rejection(host_m['d'], batch_size=10000, seed=1).sample(300, quantile=0.01,
                                                                          bar=False)
    m, dp = mg1.get_device_model(seed_obs=2)
    assert np.array_equal(m.observed['MG1'], host_m.observed['MG1'])
    res_d = elfi.Rejection(m['d'], batch_size=100000, seed=1).sample(3000, quantile=0.01, bar=False)
    s = res_d.samples
    assert np.all((s['t2'] >= s['t1']) & (s['t2'] <= s['t1'] + 10))
    for name in ('t1', 't2', 't3'):
        h, d = res_h.samples[name], res_d.samples[name]
        se = np.sqrt(h.var() / len(h) + d.var() / len(d))
        assert abs(h.mean() - d.mean()) < 4 * se, (name, h.mean(), d.mean(), se)


# ---------------------------------------------------------------------------- samplers
def test_device_model_smc_and_adaptive_distance_smc():
    import elfi_b200 as elfi
    from elfi_b200.examples import mg1
    m, dp = mg1.get_device_model(seed_obs=3)

    def in_support(s):
        return np.all((s['t1'] >= 0) & (s['t1'] <= 10) & (s['t2'] >= s['t1']) &
                      (s['t2'] <= s['t1'] + 10) & (s['t3'] >= 0) & (s['t3'] <= 0.5))

    def run(**kw):
        return elfi.SMC(m['d'], batch_size=10000, seed=4, device_proposal=dp, **kw).sample(
            1000, quantiles=[0.1, 0.3, 0.3], bar=False)
    smc = run()
    assert len(smc.populations) == 3 and np.all(np.isfinite(smc.weights))
    assert in_support(smc.samples)
    par = run(distributed=False, max_parallel_batches=2)
    par2 = run(distributed=False, max_parallel_batches=2)
    assert np.array_equal(par.samples_array, par2.samples_array)
    assert np.array_equal(par.weights, par2.weights)
    m['d'].become(elfi.AdaptiveDistance(m['quantiles']))
    ad = elfi.AdaptiveDistanceSMC(m['d'], batch_size=10000, seed=5, device_proposal=dp).sample(
        1000, rounds=3, quantile=0.3, bar=False)
    assert len(ad.populations) == 3
    assert np.all(np.isfinite(ad.samples_array)) and in_support(ad.samples)
