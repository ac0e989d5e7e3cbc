"""Device toad simulator and summaries.

* per-element replay against the kernel's own previous day (tests/toad_replay.py over
  oracle/streams.py): return decisions, refuge days and returned positions exact, non-returned
  steps within the bound of the transcendentals' ulps carried through SciPy's formula with the
  condition numbers of its two sums; row counters across 2^32; split launches equal one launch;
* toad_summaries equals NumPy bit for bit in the count, the median and the gaps before the log;
  the logs are within 2 ulp of NumPy's; strided views, the crafted goldens and both median paths;
* the fused simulator equals the unfused chain bit for bit up to B = 100003;
* statistics against the host simulator, Rejection posteriors, and the samplers.
"""
import numpy as np
import pytest
import scipy.stats as ss

import toad_replay as tr
from conftest import load_golden

pytestmark = pytest.mark.gpu
P11 = np.linspace(0, 1, 11)


def _np(t):
    return t.cpu().numpy()


def _host(x, lag, p=P11, thd=10):
    from elfi_b200.examples import toad
    with np.errstate(all='ignore'):
        return toad.compute_summaries(x, lag, p=p, thd=thd)


def _params(B, seed):
    rs = np.random.RandomState(seed)
    P = np.column_stack([rs.uniform(1, 2, B), rs.uniform(0, 100, B), rs.uniform(0, 0.9, B)])
    corners = np.array([[1.0, 0.0, 0.0], [1.0, 100.0, 0.9], [2.0, 0.0, 0.9], [2.0, 100.0, 0.0],
                        [1.0, 35.0, 0.0], [1.7, 35.0, 0.6]])
    P[:min(B, 6)] = corners[:min(B, 6)]
    return P


def _close(dev_s, host_s):
    """Columns 0 and 1 bit for bit; the log gaps within 2 ulp (the device's log against NumPy's)."""
    assert np.array_equal(dev_s[:, :2], host_s[:, :2])
    a, b = dev_s[:, 2:], host_s[:, 2:]
    same = (a == b) | (np.isnan(a) & np.isnan(b))
    near = np.abs(a - b) <= 2 * np.spacing(np.abs(b))
    assert np.all(same | near), np.argwhere(~(same | near))[:5]
    return int(np.sum(~same))


# ---------------------------------------------------------------------------- trajectories
@pytest.mark.parametrize('offset', [0, 2 ** 32 - 100])
def test_replay_every_toad_day(offset):
    from elfi_b200 import ops
    P = _params(300, 7)
    n_toads, n_days = 66, 63
    X, _ = ops.sim_toad(P, seed=11, offset=offset, want_data=True, lags=None)
    X = _np(X)                                                  # (B, n_days, n_toads)
    assert np.all(X[:, 0] == 0)
    u_ret, word, u_th, u_w = tr.draws(len(P), n_toads, n_days, 11, offset)
    alpha, gamma, p0 = (P[:, j][:, None] for j in range(3))
    worst_c = 0.0
    for d in range(1, n_days):
        ret = u_ret[:, d - 1] < p0
        j = tr.refuge_day(word[:, d - 1], d)
        back = np.take_along_axis(X, j[:, None, :], axis=1)[:, 0]
        assert np.array_equal(X[:, d][ret], back[ret], equal_nan=True), d
        s, c1, c2 = tr.step(np.broadcast_to(alpha, ret.shape), np.broadcast_to(gamma, ret.shape),
                            u_th[:, d - 1], u_w[:, d - 1])
        want = X[:, d - 1] + s
        bound = tr.step_bound(s, np.broadcast_to(alpha, ret.shape), c1, c2) + \
            2 * np.spacing(np.abs(want))
        nr = ~ret
        fin = nr & np.isfinite(want)
        assert np.all(np.abs(X[:, d] - want)[fin] <= bound[fin]), d
        assert np.array_equal(np.isnan(X[:, d][nr]), np.isnan(want[nr])), d
        cc = np.maximum(c1, c2)[nr & (np.broadcast_to(alpha, ret.shape) > 1)]
        worst_c = max(worst_c, float(cc[np.isfinite(cc)].max(initial=0.0)))
    # beta = 0: the sums cancel at most by 1 / cos((alpha - 1) pi / 2), large only as alpha -> 2
    print('largest condition number of the two sums: %.3g' % worst_c)
    # alpha == 1 and gamma == 0 (row 0): NaN steps, as in SciPy
    assert np.isnan(X[0, 1:]).any()


def test_split_launches_equal_one_launch():
    from elfi_b200 import ops
    P = _params(1000, 3)
    base = 2 ** 32 - 400
    whole = ops.sim_toad(P, seed=9, offset=base, want_data=True)
    fused = ops.sim_toad(P, seed=9, offset=base)[1]
    assert np.array_equal(_np(whole[1]), _np(fused), equal_nan=True)
    for cut in (1, 400, 777):
        parts = [ops.sim_toad(P[:cut], seed=9, offset=base, want_data=True),
                 ops.sim_toad(P[cut:], seed=9, offset=base + cut, want_data=True)]
        for j in range(2):
            joined = np.concatenate([_np(parts[0][j]), _np(parts[1][j])])
            assert np.array_equal(joined, _np(whole[j]), equal_nan=True), (cut, j)


def test_invalid_parameters_give_nan_rows():
    from elfi_b200 import ops
    P = np.array([[2.5, 10.0, 0.5], [0.0, 10.0, 0.5], [1.5, -1.0, 0.5], [np.nan, 1.0, 0.5],
                  [1.5, 10.0, 0.5]])
    X, S = ops.sim_toad(P, want_data=True)
    X, S = _np(X), _np(S)
    assert np.isnan(X[:4]).all() and np.isfinite(X[4]).all()
    assert np.array_equal(S[:4], np.tile(np.r_[0.0, np.full(11, np.inf)], (4, 4)))


# ---------------------------------------------------------------------------- summaries
@pytest.mark.parametrize('n_toads,n_days,lag', [(66, 63, 1), (66, 63, 2), (66, 63, 4), (66, 63, 8),
                                                (5, 9, 3), (54, 12, 1), (55, 12, 1), (1, 2, 1),
                                                (4092, 2, 1), (2, 2049, 1)])
def test_summaries_equal_numpy(n_toads, n_days, lag):
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    rs = np.random.RandomState(n_toads * 7 + n_days)
    B = 200
    x = np.cumsum(rs.standard_cauchy((n_days, n_toads, B)) * 20, axis=0)
    x[:, :, 1] = 0.0
    x[1, 0, 2] = np.nan
    x[-1, -1, 3] = np.inf
    x[:, :, 4] = np.round(x[:, :, 4] / 50) * 50       # ties
    want = _host(x, lag)
    n_log = _close(_np(ops.toad_summaries(x, lag)), want)
    big = dev.to_device(rs.standard_normal((n_days + 1, n_toads + 2, 2 * B)))
    big[1:, 1:n_toads + 1, ::2] = dev.to_device(x)
    view = big[1:, 1:n_toads + 1, ::2]
    assert np.array_equal(_np(ops.toad_summaries(view, lag)), _np(ops.toad_summaries(x, lag)))
    p, thd = np.array([0.9, 0.1, 0.5, 1.0]), 2.5
    _close(_np(ops.toad_summaries(x, lag, p=p, thd=thd)), _host(x, lag, p=p, thd=thd))
    print('%d of %d log gaps differ from NumPy (within 2 ulp)' % (n_log, want[:, 2:].size))


def test_summaries_of_crafted_goldens():
    from elfi_b200 import ops
    g = load_golden('toad_summaries')
    for n in [k[2:] for k in g if k.startswith('x_')]:
        got = _np(ops.toad_summaries(g['x_' + n], int(g['lag_' + n]), p=g['p_' + n],
                                     thd=float(g['thd_' + n])))
        _close(got, g['s_' + n])
    draws = load_golden('toad_draws')
    for lag in range(1, 9):
        _close(_np(ops.toad_summaries(draws['x'], lag)), g['draws_lag{}'.format(lag)])


@pytest.mark.parametrize('B', [1, 2, 31, 100003])
def test_fused_equals_unfused_chain(B):
    from elfi_b200 import ops
    P = _params(B, B % 97)
    X, S_chain = ops.sim_toad(P, seed=5, offset=2 ** 32 - B // 2, want_data=True)
    _, S = ops.sim_toad(P, seed=5, offset=2 ** 32 - B // 2)
    S, S_chain = _np(S), _np(S_chain)
    assert np.array_equal(S, S_chain)
    xr = X.permute(1, 2, 0)
    for j, lag in enumerate((1, 2, 4, 8)):
        assert np.array_equal(_np(ops.toad_summaries(xr, lag)), S[:, 12 * j:12 * (j + 1)])
    rows = np.unique(np.linspace(0, B - 1, min(B, 100)).astype(int))
    host_x = _np(xr[:, :, rows])
    for j, lag in enumerate((1, 2, 4, 8)):
        _close(S[rows, 12 * j:12 * (j + 1)], _host(host_x, lag))


# ---------------------------------------------------------------------------- statistics
@pytest.mark.parametrize('prm', [(1.7, 35.0, 0.6), (1.2, 10.0, 0.2), (1.95, 80.0, 0.85)])
def test_statistics_match_host_simulator(prm):
    from elfi_b200 import ops
    from elfi_b200.examples import toad
    n_host = 1500
    xh = toad.toad(*prm, batch_size=n_host, random_state=np.random.RandomState(1))
    _, S = ops.sim_toad(np.tile(prm, (40000, 1)), seed=77)
    S = _np(S)
    for j, lag in enumerate((1, 2, 4, 8)):
        host = _host(xh, lag)
        for c in range(12):
            dv, hv = S[:, 12 * j + c], host[:, c]
            if np.all(hv == hv[0]) and np.all(dv == hv[0]):
                continue
            assert ss.ks_2samp(dv, hv).pvalue > 1e-4, (prm, lag, c)


def test_device_rejection_posterior_matches_host():
    import elfi_b200 as elfi
    from elfi_b200.examples import toad
    host_m = toad.get_model(seed_obs=2)
    res_h = elfi.Rejection(host_m['d'], batch_size=1000, seed=1).sample(40, quantile=0.01,
                                                                        bar=False)
    m, dp = toad.get_device_model(seed_obs=2)
    assert np.array_equal(m.observed['toad'], host_m.observed['toad'])
    res_d = elfi.Rejection(m['d'], batch_size=100000, seed=1).sample(2000, quantile=0.01, bar=False)
    for name in ('alpha', 'gamma', 'p0'):
        h, d = res_h.samples[name], res_d.samples[name]
        se = np.sqrt(h.var() / len(h) + d.var() / len(d))
        assert abs(h.mean() - d.mean()) < 4 * se, (name, h.mean(), d.mean(), se)


def test_device_model_rejection_and_smc():
    import elfi_b200 as elfi
    from elfi_b200.examples import toad
    m, dp = toad.get_device_model(seed_obs=3)
    res = elfi.Rejection(m['d'], batch_size=20000, seed=1).sample(200, quantile=0.01, bar=False)
    assert res.n_samples == 200 and not np.any(np.isnan(res.discrepancies))

    def run(**kw):
        return elfi.SMC(m['d'], batch_size=10000, seed=4, device_proposal=dp, **kw).sample(
            500, quantiles=[0.1, 0.3, 0.3], bar=False)
    smc = run()
    assert len(smc.populations) == 3 and np.all(np.isfinite(smc.weights))
    par = run(distributed=False, max_parallel_batches=2)
    par2 = run(distributed=False, max_parallel_batches=2)
    assert np.array_equal(par.samples_array, par2.samples_array)
    assert np.array_equal(par.weights, par2.weights)
