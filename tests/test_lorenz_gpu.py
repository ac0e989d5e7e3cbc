"""Device Lorenz simulator and summaries.

* phi = 1 (eta stays exactly 0): whole device trajectories equal the NumPy restatement bit for bit at
  every step, for ring sizes that cover every lane layout (V = 1, 2, 4 variables per lane) and a
  partial last lane;
* phi = 0 (eta is the raw normal) and the default phi (the AR(1) replayed): every step equals the
  NumPy RK4 step from the kernel's own y_{s-1} with the normals replayed through oracle/streams.py
  (tests/lorenz_replay.py), within a bound from the normals' ulps; row counters across 2^32, split
  launches equal one launch bit for bit;
* lorenz_summaries equals NumPy bit for bit, including strided, unaligned and NaN / inf rows; the
  fused simulator equals the unfused chain bit for bit;
* statistics against the host forecast_lorenz, Rejection posteriors, and the samplers.
"""
import numpy as np
import pytest
import scipy.stats as ss

import lorenz_replay as lr

pytestmark = pytest.mark.gpu
DT = 4 / 160


def _np(t):
    return t.cpu().numpy()


def _host_summaries(x):
    from elfi_b200.examples import lorenz
    with np.errstate(all='ignore'):
        return np.column_stack([lorenz.mean(x), lorenz.var(x), lorenz.autocov(x), lorenz.cov(x),
                                lorenz.xcov(x, True), lorenz.xcov(x, False)])


def _init(m):
    from elfi_b200.examples import lorenz
    return np.array(lorenz.INITIAL_STATE) if m == 40 else np.random.RandomState(m).randn(m) * 4


def _params(B, seed):
    rs = np.random.RandomState(seed)
    P = np.column_stack([rs.uniform(0.5, 3.5, B), rs.uniform(0, 0.3, B)])
    corners = np.array([[0.5, 0.0], [0.5, 0.3], [3.5, 0.0], [3.5, 0.3]])
    P[:4] = corners[:min(B, 4)]
    return P


# ---------------------------------------------------------------------------- trajectories
@pytest.mark.parametrize('m', [4, 5, 40, 41, 65, 67, 128])
def test_noise_free_trajectories_equal_numpy(m):
    from elfi_b200 import ops
    P = _params(37, m)
    init = _init(m)
    X, _ = ops.sim_lorenz(P, initial_state=init, phi=1.0, seed=3, want_data=True,
                          want_summaries=False)
    X = _np(X)
    y = np.tile(init, (len(P), 1))
    assert np.array_equal(X[:, 0], y)
    with np.errstate(all='ignore'):
        for s in range(1, 160):
            y = lr.rk4_step(y, np.zeros_like(y), P[:, 0], P[:, 1], 10.0, DT)
            assert np.array_equal(X[:, s], y, equal_nan=True), (m, s)


def _one_step_checks(X, P, T, seed, offset, phi):
    B, _, m = X.shape
    e, err = lr.normals(B, T, m, seed, offset)
    s_phi = float(np.sqrt(1 - pow(phi, 2)))
    eta, eb = lr.eta_replay(e, err, phi, s_phi)
    with np.errstate(all='ignore'):
        for s in range(1, T):
            want = lr.rk4_step(X[:, s - 1], eta[:, s - 1], P[:, 0], P[:, 1], 10.0, DT)
            bound = lr.one_step_bound(want, eb[:, s - 1], DT)
            ok = np.abs(X[:, s] - want) <= bound
            assert ok.all(), (s, np.argwhere(~ok)[:5], np.max(np.abs(X[:, s] - want)))


@pytest.mark.parametrize('phi', [0.0, 0.984])
@pytest.mark.parametrize('offset', [0, 2 ** 32 - 150])
def test_one_step_replay(phi, offset):
    from elfi_b200 import ops
    P = _params(300, 7)
    X, _ = ops.sim_lorenz(P, phi=phi, seed=11, offset=offset, want_data=True, want_summaries=False)
    X = _np(X)
    assert np.isfinite(X).all()
    _one_step_checks(X, P, 160, 11, offset, phi)


@pytest.mark.parametrize('m', [5, 41, 67])
def test_one_step_replay_other_layouts(m):
    from elfi_b200 import ops
    P = _params(100, m)
    # total_duration 1 keeps the step at DT = 4 / 160
    X, _ = ops.sim_lorenz(P, n_timestep=40, initial_state=_init(m), phi=0.0, total_duration=1.0,
                          seed=2, offset=2 ** 32 - 50, want_data=True, want_summaries=False)
    _one_step_checks(_np(X), P, 40, 2, 2 ** 32 - 50, 0.0)


def test_split_launches_equal_one_launch():
    from elfi_b200 import ops
    P = _params(1000, 3)
    base = 2 ** 32 - 400
    whole = ops.sim_lorenz(P, seed=9, offset=base, want_data=True)
    fused = ops.sim_lorenz(P, seed=9, offset=base)[1]
    assert np.array_equal(_np(whole[1]), _np(fused), equal_nan=True)
    for cut in (1, 400, 777):
        parts = [ops.sim_lorenz(P[:cut], seed=9, offset=base, want_data=True),
                 ops.sim_lorenz(P[cut:], seed=9, offset=base + cut, want_data=True)]
        for j in range(2):
            joined = np.concatenate([_np(parts[0][j]), _np(parts[1][j])])
            assert np.array_equal(joined, _np(whole[j]), equal_nan=True), (cut, j)


def test_phi_above_one_gives_nan_rows():
    from elfi_b200 import ops
    X, S = ops.sim_lorenz(_params(5, 1), n_timestep=4, phi=1.5, want_data=True)
    X = _np(X)
    assert np.isfinite(X[:, 0]).all() and np.isnan(X[:, 1:]).all() and np.isnan(_np(S)).all()


# ---------------------------------------------------------------------------- bit-for-bit summaries
@pytest.mark.parametrize('T,m', [(2, 4), (3, 5), (17, 7), (160, 40), (161, 40), (159, 64), (160, 128),
                                 (9, 2), (17, 3), (240, 128)])
def test_summaries_equal_numpy(T, m):
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    rs = np.random.RandomState(T * 1000 + m)
    B = 500
    x = rs.randn(B, T, m) * 10 ** rs.uniform(-2, 2, (B, 1, 1))
    x[1, T // 2, m // 2] = np.nan
    x[2, 0, 0] = np.inf
    x[3, -1, -1], x[3, 0, -1] = -np.inf, np.inf
    x[4] = 2.5
    x[5] = -0.0
    want = _host_summaries(x)
    assert np.array_equal(_np(ops.lorenz_summaries(x)), want, equal_nan=True)
    c0 = 1 if (m + 4) % 2 else 2                 # an odd element offset: an unaligned view
    big = dev.to_device(np.concatenate([rs.randn(B, 1, m + 3), np.concatenate(
        [rs.randn(B, T, c0), x, rs.randn(B, T, 3 - c0)], axis=2), rs.randn(B, 1, m + 3)], axis=1))
    view = big[:, 1:T + 1, c0:c0 + m]
    assert view.data_ptr() % 16 != 0
    assert np.array_equal(_np(ops.lorenz_summaries(view)), want, equal_nan=True)
    tr = dev.to_device(np.ascontiguousarray(x.transpose(0, 2, 1))).transpose(1, 2)   # ld_k = T
    assert np.array_equal(_np(ops.lorenz_summaries(tr)), want, equal_nan=True)


@pytest.mark.parametrize('B', [1, 2, 3, 31, 100003])
def test_fused_equals_unfused_chain(B):
    from elfi_b200 import ops
    P = _params(B, B % 97)
    X, S_chain = ops.sim_lorenz(P, seed=5, offset=2 ** 32 - B // 2, want_data=True)
    _, S = ops.sim_lorenz(P, seed=5, offset=2 ** 32 - B // 2)
    S, S_chain = _np(S), _np(S_chain)
    assert np.array_equal(S, S_chain, equal_nan=True)
    assert np.array_equal(_np(ops.lorenz_summaries(X)), S, equal_nan=True)
    rows = np.unique(np.linspace(0, B - 1, min(B, 200)).astype(int))
    assert np.array_equal(_host_summaries(_np(X[rows])), S[rows], equal_nan=True)
    assert np.isfinite(S).all()


@pytest.mark.parametrize('m', [4, 41, 67, 128])
def test_fused_equals_unfused_other_layouts(m):
    from elfi_b200 import ops
    P = _params(1001, m)
    init = _init(m)
    X, S_chain = ops.sim_lorenz(P, n_timestep=100, initial_state=init, seed=4, want_data=True)
    _, S = ops.sim_lorenz(P, n_timestep=100, initial_state=init, seed=4)
    assert np.array_equal(_np(S), _np(S_chain), equal_nan=True)
    assert np.array_equal(_host_summaries(_np(X)), _np(S), equal_nan=True)


def test_observed_summaries_on_device_equal_host():
    from elfi_b200 import device as dev
    from elfi_b200.examples import lorenz
    m, _ = lorenz.get_device_model(seed_obs=2)
    obs = np.asarray(m.observed['Lorenz'])
    fns = (lorenz.mean, lorenz.var, lorenz.autocov, lorenz.cov, lambda x: lorenz.xcov(x, True),
           lambda x: lorenz.xcov(x, False))
    for f in fns:
        assert np.array_equal(_np(f(dev.to_device(obs))), f(obs))


# ---------------------------------------------------------------------------- statistics
def test_statistics_match_host_simulator():
    from elfi_b200 import ops
    from elfi_b200.examples import lorenz
    n_host = 10000
    xh = lorenz.forecast_lorenz(2.0, 0.1, batch_size=n_host, random_state=np.random.RandomState(1))
    host = _host_summaries(xh)
    _, S = ops.sim_lorenz(np.tile([2.0, 0.1], (50000, 1)), seed=77)
    S = _np(S)
    for j in range(6):
        assert ss.ks_2samp(S[:, j], host[:, j]).pvalue > 1e-3, j


def test_device_rejection_posterior_matches_host():
    import elfi_b200 as elfi
    from elfi_b200.examples import lorenz
    host_m = lorenz.get_model(seed_obs=2)
    res_h = elfi.Rejection(host_m['d'], batch_size=2000, seed=1).sample(100, quantile=0.01,
                                                                        bar=False)
    m, dp = lorenz.get_device_model(seed_obs=2)
    assert np.array_equal(m.observed['Lorenz'], host_m.observed['Lorenz'])
    res_d = elfi.Rejection(m['d'], batch_size=100000, seed=1).sample(3000, quantile=0.01, bar=False)
    for name in ('theta1', 'theta2'):
        h, d = res_h.samples[name], res_d.samples[name]
        se = np.sqrt(h.var() / len(h) + d.var() / len(d))
        assert abs(h.mean() - d.mean()) < 4 * se, (name, h.mean(), d.mean(), se)


# ---------------------------------------------------------------------------- samplers
def test_device_model_rejection_and_smc():
    import elfi_b200 as elfi
    from elfi_b200.examples import lorenz
    m, dp = lorenz.get_device_model(seed_obs=3)
    res = elfi.Rejection(m['d'], batch_size=20000, seed=1).sample(200, quantile=0.01, bar=False)
    assert res.n_samples == 200 and not np.any(np.isnan(res.discrepancies))
    assert abs(res.sample_means['theta1'] - 2.0) < 0.5

    def run(**kw):
        return elfi.SMC(m['d'], batch_size=10000, seed=4, device_proposal=dp, **kw).sample(
            1000, quantiles=[0.1, 0.3, 0.3], bar=False)
    smc = run()
    assert len(smc.populations) == 3 and np.all(np.isfinite(smc.weights))
    par = run(distributed=False, max_parallel_batches=2)
    par2 = run(distributed=False, max_parallel_batches=2)
    assert np.array_equal(par.samples_array, par2.samples_array)
    assert np.array_equal(par.weights, par2.weights)
