"""Device Lotka-Volterra simulator and summaries.

* per-row replay (tests/lv_replay.py over oracle/streams.py): event counts and observations equal
  the kernel's exactly, except where the replay finds an event time within 1e-12 (relative) of a
  grid time or of time_end, or a noisy value within 1e-12 of an integer (the device's log and
  Box-Muller against NumPy's); also for capped rows, invalid rows, row counters across 2^32, a batch
  that is not a multiple of 32, and split launches against one launch;
* lv_summaries equals NumPy bit for bit but for the log (within 1 ulp), on strided views too;
* statistics against the host simulator, Rejection posteriors, and SMC determinism.
Every simulator call passes a small max_events, which bounds its run time.
"""
import numpy as np
import pytest
import scipy.stats as ss

import lv_replay

pytestmark = pytest.mark.gpu
TRUTH = [1.0, 0.005, 0.6, 50, 100, 0.]
MARGIN = 1e-12


def _np(t):
    return t.cpu().numpy()


def _summ(x):
    from elfi_b200.examples import lotka_volterra as lv
    with np.errstate(all='ignore'):
        return np.column_stack([
            lv.stock_mean(x, 0), lv.stock_mean(x, 1), lv.stock_log_variance(x, 0),
            lv.stock_log_variance(x, 1), lv.stock_autocorr(x, 0, 1), lv.stock_autocorr(x, 1, 1),
            lv.stock_autocorr(x, 0, 2), lv.stock_autocorr(x, 1, 2), lv.stock_crosscorr(x)])


def _prior_params(B, seed, noise=False):
    rs = np.random.RandomState(seed)
    P = np.column_stack([np.exp(rs.uniform(-6, 2, (B, 3))), rs.normal(50, np.sqrt(50), B),
                         rs.normal(100, 10, B),
                         np.exp(rs.uniform(np.log(0.5), np.log(50), B)) if noise else np.zeros(B)])
    return P


def _check_replay(P, n_obs, time_end, seed, offset, max_events):
    from elfi_b200 import ops
    obs, n = ops.sim_lotka_volterra(P, n_obs, time_end, seed=seed, offset=offset,
                                    max_events=max_events)
    obs, n = _np(obs), _np(n)
    want, kw, margin = lv_replay.simulate(P, n_obs, time_end, seed, offset, max_events)
    same = (n == kw) & np.all((obs == want) | (np.isnan(obs) & np.isnan(want)), axis=(1, 2))
    excused = ~same & (margin <= MARGIN)
    print('rows %d, differing %d (all within %.0e of a grid time or integer), smallest margin '
          '%.3g' % (len(P), int((~same).sum()), MARGIN, float(margin.min())))
    assert np.all(same | excused), (np.nonzero(~same & ~excused)[0][:5], margin[~same])
    return obs, n


@pytest.mark.parametrize('offset', [0, 2 ** 32 - 20])
def test_replay_prior_rows(offset):
    P = _prior_params(45, 1)
    P[:3] = TRUTH
    obs, n = _check_replay(P, 30, 30.0, 11, offset, 20000)
    assert np.isfinite(obs[:3]).all() and np.all(n[:3] > 100)


def test_replay_noise_truth_and_edges():
    P = np.array([TRUTH, [1.0, 0.005, 0.6, 3.0, 2.0, 10.0], [0.3, 0.01, 1.0, 1.0, 1.0, 25.0],
                  [0.1, 0.02, 1.5, 30.0, 12.0, 0.], [1.0, 0.005, 0.6, 40.0, 0.5, 0.],
                  [0.7, 0.005, 0.6, 0.3, 0.2, 0.], [1.0, 0.005, 0.6, 0.0, 30.0, 2.0]] * 5)
    P[::5, 5] = 5.0
    obs, n = _check_replay(P, 50, 30.0, 4, 2 ** 32 - 7, 50000)
    assert (obs < 0).any() and np.isfinite(obs).all()


def test_capped_and_invalid_rows():
    P = np.array([TRUTH, TRUTH, [-1.0, 0.005, 0.6, 50, 100, 0.], [1.0, np.nan, 0.6, 50, 100, 0.],
                  [1.0, 0.005, 0.6, -3.0, 100, 0.], [1.0, 0.005, 0.6, 50, 2.0 ** 31, 0.],
                  [1.0, 0.005, 0.6, 50, 100, -1.0], [1.0, 0.005, 0.6, 50, 100, np.nan],
                  [np.inf, 0.005, 0.6, 50, 100, 0.]])
    obs, n = _check_replay(P, 16, 30.0, 3, 0, 300)
    assert np.isnan(obs).all() and np.all(n[:2] == 300) and np.all(n[2:8] == 0)
    assert n[8] == 300


@pytest.mark.parametrize('B', [1, 31, 33, 100])
def test_split_launches_equal_one_launch(B):
    from elfi_b200 import ops
    P = _prior_params(B, B)
    P[: B // 2] = TRUTH
    base = 2 ** 32 - B // 2
    whole = ops.sim_lotka_volterra(P, 20, 30.0, seed=9, offset=base, max_events=30000)
    for cut in sorted({0, 1, B // 3, B - 1}):
        parts = [ops.sim_lotka_volterra(P[:cut], 20, 30.0, seed=9, offset=base, max_events=30000),
                 ops.sim_lotka_volterra(P[cut:], 20, 30.0, seed=9, offset=base + cut,
                                        max_events=30000)]
        for j in range(2):
            joined = np.concatenate([_np(parts[0][j]), _np(parts[1][j])])
            assert np.array_equal(joined, _np(whole[j]), equal_nan=True), (cut, j)
    if B == 100:
        rows = np.r_[0:3, 50:60]
        _check_replay(P[rows], 20, 30.0, 9, 0, 30000)


# ---------------------------------------------------------------------------- summaries
def _close(dev_s, host_s):
    """Bit for bit but for the log columns 2, 3, within 1 ulp."""
    keep = [0, 1, 4, 5, 6, 7, 8]
    assert np.array_equal(dev_s[:, keep], host_s[:, keep], equal_nan=True)
    a, b = dev_s[:, 2:4], host_s[:, 2:4]
    same = (a == b) | (np.isnan(a) & np.isnan(b))
    assert np.all(same | (np.abs(a - b) <= np.spacing(np.abs(b)))), np.argwhere(~same)[:5]
    return int((~same).sum())


def test_summaries_equal_numpy_on_device_output():
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    P = _prior_params(3000, 5)
    P[:1000] = TRUTH
    obs, _ = ops.sim_lotka_volterra(P, 50, 30.0, seed=2, max_events=20000)
    host = _np(obs)
    n_log = _close(_np(ops.lv_summaries(obs)), _summ(host))
    print('%d of %d log summaries differ from NumPy by an ulp' % (n_log, 2 * len(P)))
    rs = np.random.RandomState(3)
    for n_obs in (3, 4, 7, 8, 9, 16, 50, 127, 128):
        x = rs.randint(-100, 5000, (257, n_obs, 2)).astype(np.float64)
        x[0] = 5.0
        x[1, :, 1] = 0.0
        big = dev.to_device(rs.standard_normal((2 * 257, n_obs + 3, 5)))
        big[::2, 1:n_obs + 1, 1:5:2] = dev.to_device(x)
        view = big[::2, 1:n_obs + 1, 1:5:2]
        want = _summ(x)
        _close(_np(ops.lv_summaries(view)), want)
        assert np.array_equal(_np(ops.lv_summaries(view)), _np(ops.lv_summaries(x)), equal_nan=True)


# ---------------------------------------------------------------------------- statistics
@pytest.mark.parametrize('prm', [TRUTH, [0.5, 0.05, 3.0, 10.0, 4.0, 0.],
                                 [1.0, 0.005, 0.6, 50, 100, 10.0]])
def test_statistics_match_host_simulator(prm):
    from elfi_b200 import ops
    from elfi_b200.examples import lotka_volterra as lv
    xh = lv.lotka_volterra(*prm, n_obs=50, batch_size=600, random_state=np.random.RandomState(1))
    obs, n = ops.sim_lotka_volterra(np.tile(prm, (20000, 1)), 50, 30.0, seed=77, max_events=200000)
    assert np.all(_np(n) < 200000)
    host, dv = _summ(xh), _np(ops.lv_summaries(obs))
    for c in range(9):
        d, h = dv[:, c], host[:, c]
        d, h = d[np.isfinite(d)], h[np.isfinite(h)]
        if h.size and np.all(h == h[0]) and np.all(d == h[0]):
            continue
        assert ss.ks_2samp(d, h).pvalue > 1e-4, (prm, c)
    for j in (1, 10, 30, 49):
        for s in (0, 1):
            assert ss.ks_2samp(_np(obs)[:, j, s], xh[:, j, s]).pvalue > 1e-4, (prm, j, s)


def test_device_rejection_posterior_matches_host():
    import elfi_b200 as elfi
    from elfi_b200.examples import lotka_volterra as lv
    host_m = lv.get_model(n_obs=20, seed_obs=2, time_end=2.0)
    res_h = elfi.Rejection(host_m['d'], batch_size=100, seed=1).sample(40, quantile=0.05,
                                                                       bar=False)
    m, dp = lv.get_device_model(n_obs=20, seed_obs=2, time_end=2.0, max_events=200000)
    assert np.array_equal(m.observed['LV'], host_m.observed['LV'])
    res_d = elfi.Rejection(m['d'], batch_size=100000, seed=1).sample(5000, quantile=0.05, bar=False)
    for name in dp.parameter_names:
        h, d = np.log(res_h.samples[name]) if name[0] == 'r' else res_h.samples[name], \
            np.log(res_d.samples[name]) if name[0] == 'r' else res_d.samples[name]
        se = np.sqrt(h.var() / len(h) + d.var() / len(d))
        assert abs(h.mean() - d.mean()) < 4.5 * se, (name, h.mean(), d.mean(), se)


def test_device_model_rejection_and_smc():
    import elfi_b200 as elfi
    from elfi_b200.examples import lotka_volterra as lv
    m, dp = lv.get_device_model(seed_obs=3, max_events=100000)
    res = elfi.Rejection(m['d'], batch_size=20000, seed=1).sample(200, quantile=0.01, bar=False)
    assert res.n_samples == 200 and not np.any(np.isnan(res.discrepancies))

    def run(**kw):
        return elfi.SMC(m['d'], batch_size=10000, seed=4, device_proposal=dp, **kw).sample(
            300, quantiles=[0.1, 0.3], bar=False)
    smc = run()
    assert len(smc.populations) == 2 and np.all(np.isfinite(smc.weights))
    par = run(distributed=False, max_parallel_batches=2)
    par2 = run(distributed=False, max_parallel_batches=2)
    assert np.array_equal(par.samples_array, par2.samples_array)
    assert np.array_equal(par.weights, par2.weights)
