"""Device stochastic volatility simulator.

* sim_svm element by element against the NumPy replay of its Philox streams (tests/svm_replay.py):
  the shocks within the bound of the transcendentals' ulps carried through SciPy's formula, the
  data within that bound and the log-volatility's, carried through the AR(1); NaN exactly where
  the replay has NaN; row counters across 2^32; split launches equal one launch; invalid
  parameters give NaN rows;
* the fused kurt / skew equal the unfused chain (svm_summaries) bit for bit, and NumPy's kurt /
  skew of the materialised data;
* statistics against the host simulator, the Rejection posterior against the host model's, and
  the samplers.
"""
import numpy as np
import pytest
import scipy.stats as ss

import svm_replay as sr

pytestmark = pytest.mark.gpu
FIXED = (1.0, 0.0, 0.0, 0.95, 0.2)          # kappa, eta, mu, phi, sigma
CORNERS = [(1.2, 0.5), (1.0, 0.5), (1.0, 1.0), (1.0, -1.0), (1.0, 0.0), (2.0, 0.3), (0.5, -1.0),
           (1.5, 1.0), (1.7, 0.0), (1.3, -0.0)]


def _np(t):
    return t.cpu().numpy()


def _same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True) and \
        np.array_equal(np.signbit(a[a == 0]), np.signbit(b[a == 0]))


def _params(B, rs, wide=False):
    """(B, 7): alpha, beta from the priors (the corners first); with wide, kappa, eta, mu, phi and
    sigma drawn too (kappa = 0 included), else the reference's constants."""
    P = np.empty((B, 7))
    P[:, 0], P[:, 1] = rs.uniform(0.5, 2.0, B), rs.uniform(-1, 1, B)
    P[:, 2:] = FIXED
    if wide:
        P[:, 2] = rs.uniform(0, 3, B)
        P[:, 3] = rs.uniform(-1, 1, B)
        P[:, 4] = rs.uniform(-1, 1, B)
        P[:, 5] = rs.uniform(-0.99, 0.99, B)
        P[:, 6] = rs.uniform(0, 0.5, B)
        P[len(CORNERS):len(CORNERS) + 10, 2] = 0.0
    P[:len(CORNERS), :2] = CORNERS
    return P


# ---------------------------------------------------------------------------- streams and bounds
def test_uniforms_and_shocks_match_replay():
    """With mu = sigma = 0 the log-volatility is 0 and y is the shock itself: every shock within
    the bound carried through SciPy's formula, NaN exactly where the replay has NaN."""
    from elfi_b200 import ops
    rs = np.random.RandomState(3)
    B, n = 4000, 50
    P = _params(B, rs, wide=True)
    P[:, 4], P[:, 6] = 0.0, 0.0
    offset = 2 ** 32 - 1500
    Y, _ = ops.sim_svm(P, n, seed=5, offset=offset, want_data=True, want_summaries=False)
    Y = _np(Y)
    _, _, v, v_err, x, cond = sr.sim_svm(P, n, seed=5, offset=offset)
    assert np.all(x == 0)
    assert np.array_equal(np.isnan(Y), np.isnan(v))
    fin = np.isfinite(v)
    bad = fin & ~(np.abs(Y - v) <= v_err)
    assert not bad.any(), (np.argwhere(bad)[:5], (Y - v)[bad][:5], v_err[bad][:5])
    # a wrong stream would be O(1) off: the bound is tight enough to tell
    assert np.median(v_err[fin] / np.maximum(np.abs(v[fin]), 1e-300)) < 1e-12
    print('largest condition number of the denominator and numerator sums: %.3g' %
          cond[np.isfinite(cond)].max())
    # kappa == 0 off alpha == 1: the shocks are eta exactly
    z = (P[:, 2] == 0) & (P[:, 0] != 1)
    assert np.array_equal(Y[z], np.broadcast_to(P[z, 3:4], Y[z].shape))


@pytest.mark.parametrize('offset', [0, 2 ** 32 - 300])
@pytest.mark.parametrize('n_obs', [2, 7, 50, 512])
def test_sim_svm_matches_replay(offset, n_obs):
    from elfi_b200 import ops
    rs = np.random.RandomState(n_obs + offset % 89)
    B = 1000
    P = _params(B, rs, wide=n_obs != 50)
    Y, _ = ops.sim_svm(P, n_obs, seed=7, offset=offset, want_data=True, want_summaries=False)
    Y = _np(Y)
    want, err, _, _, _, _ = sr.sim_svm(P, n_obs, seed=7, offset=offset)
    assert np.array_equal(np.isnan(Y), np.isnan(want))
    fin = np.isfinite(want)
    bad = fin & ~(np.abs(Y - want) <= err)
    assert not bad.any(), (np.argwhere(bad)[:5], np.abs(Y - want)[bad][:5], err[bad][:5])
    assert np.median(err[fin] / np.maximum(np.abs(want[fin]), 1e-300)) < 1e-11


def test_split_launches_equal_one_launch():
    from elfi_b200 import ops
    P = _params(1000, np.random.RandomState(2))
    base = 2 ** 32 - 400
    whole = ops.sim_svm(P, 50, seed=9, offset=base, want_data=True)
    for cut in (1, 400, 777):
        parts = [ops.sim_svm(P[:cut], 50, seed=9, offset=base, want_data=True),
                 ops.sim_svm(P[cut:], 50, seed=9, offset=base + cut, want_data=True)]
        for j in range(2):
            joined = np.concatenate([_np(parts[0][j]), _np(parts[1][j])])
            assert _same_bits(joined, _np(whole[j])), (cut, j)


def test_invalid_parameters_give_nan_rows():
    from elfi_b200 import ops
    ok = (1.2, 0.5) + FIXED
    bad = [(0.0, 0.5), (2.5, 0.5), (np.nan, 0.5), (1.2, 1.5), (1.2, -1.5), (1.2, np.nan)]
    P = [b + FIXED for b in bad]
    P += [(1.2, 0.5, -1.0, 0, 0, 0.95, 0.2), (1.2, 0.5, np.nan, 0, 0, 0.95, 0.2),
          (1.2, 0.5, 1, 0, 0, 0.95, -0.2), (1.2, 0.5, 1, 0, 0, np.nan, 0.2),
          (1.2, 0.5, 1, 0, 0, 0.95, np.nan), ok, (1.0, 0.5, 0.0, 0, 0, 0.95, 0.2)]
    Y, S = ops.sim_svm(np.array(P), 20, seed=1, want_data=True)
    Y, S = _np(Y), _np(S)
    assert np.isnan(Y[:11]).all() and np.isnan(S[:11]).all()
    assert np.isfinite(Y[11]).all() and np.isfinite(S[11]).all()
    # kappa == 0 at alpha == 1: 0 * log(0) = NaN, as SciPy computes
    assert np.isnan(Y[12]).all()


# ---------------------------------------------------------------------------- bit-for-bit summaries
@pytest.mark.parametrize('B', [1, 129, 100003])
def test_fused_summaries_equal_unfused_chain(B):
    from elfi_b200 import ops
    from elfi_b200.examples import stochastic_volatility_model as svm
    rs = np.random.RandomState(B % 1000)
    P = _params(max(B, len(CORNERS) + 20), rs, wide=True)[:B]
    P[B // 2] = (2.5, 0.5) + FIXED
    for n_obs in (50, 512, 2, 33):
        Y, S = ops.sim_svm(P, n_obs, seed=3, offset=2 ** 32 - 1000, want_data=True)
        _, S_only = ops.sim_svm(P, n_obs, seed=3, offset=2 ** 32 - 1000)
        assert _same_bits(_np(S), _np(ops.svm_summaries(Y))), n_obs
        assert _same_bits(_np(S_only), _np(S)), n_obs
        if B <= 129:
            y = _np(Y)
            with np.errstate(all='ignore'):
                assert _same_bits(_np(S)[:, 0], svm.kurt(y)), n_obs
                assert _same_bits(_np(S)[:, 1], svm.skew(y)), n_obs


def test_summaries_equal_golden_rows():
    from elfi_b200 import ops
    from conftest import load_golden
    g = load_golden('svm_summaries')
    d = load_golden('svm_draws')
    for src, name in ((d, 'y1'), (d, 'yb'), (d, 'yx'), (g, 'crafted'), (g, 'n2')):
        S = _np(ops.svm_summaries(src[name]))
        assert np.array_equal(S[:, 0], g[name + '_kurt'], equal_nan=True), name
        assert np.array_equal(S[:, 1], g[name + '_skew'], equal_nan=True), name


# ---------------------------------------------------------------------------- statistics
@pytest.mark.parametrize('ab', [(1.2, 0.5), (1.0, 0.5), (1.0, 0.0), (1.5, 1.0), (1.5, -1.0),
                                (0.6, 0.3), (2.0, 0.0)])
def test_statistics_match_host_simulator(ab):
    from elfi_b200 import ops
    from elfi_b200.examples import stochastic_volatility_model as svm
    B = 20000
    with np.errstate(all='ignore'):
        y_h = svm.alpha_stochastic_volatility_model(*ab, *FIXED, batch_size=B,
                                                    random_state=np.random.RandomState(1))
        host = np.column_stack([svm.kurt(y_h), svm.skew(y_h)])
    P = np.tile(ab + FIXED, (B, 1))
    Y, S = ops.sim_svm(P, 50, seed=77, want_data=True)
    S, Y = _np(S), _np(Y)
    for j in range(2):
        p = ss.ks_2samp(S[:, j], host[:, j]).pvalue
        assert p > 1e-5, (ab, j, p)
    for j in (0, 17, 49):
        p = ss.ks_2samp(Y[:, j], y_h[:, j]).pvalue
        assert p > 1e-5, (ab, 'column', j, p)


def test_device_rejection_posterior_matches_host():
    import elfi_b200 as elfi
    from elfi_b200.examples import stochastic_volatility_model as svm
    host_m = svm.get_model(seed_obs=2)
    res_h = elfi.Rejection(host_m['d'], batch_size=10000, seed=1).sample(300, quantile=0.01,
                                                                          bar=False)
    m, dp = svm.get_device_model(seed_obs=2)
    assert _same_bits(m.observed['a_svm'], host_m.observed['a_svm'])
    res_d = elfi.Rejection(m['d'], batch_size=100000, seed=1).sample(3000, quantile=0.01, bar=False)
    for name in ('alpha', 'beta'):
        h, d = res_h.samples[name], res_d.samples[name]
        se = np.sqrt(h.var() / len(h) + d.var() / len(d))
        assert abs(h.mean() - d.mean()) < 4 * se, (name, h.mean(), d.mean(), se)


# ---------------------------------------------------------------------------- samplers
def test_device_model_smc_and_adaptive_distance_smc():
    import elfi_b200 as elfi
    from elfi_b200.examples import stochastic_volatility_model as svm
    m, dp = svm.get_device_model(seed_obs=3)

    def in_support(s):
        return np.all((s['alpha'] >= 0.5) & (s['alpha'] <= 2) & (s['beta'] >= -1) &
                      (s['beta'] <= 1))

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
    m['d'].become(elfi.AdaptiveDistance(m['kurt'], m['skew']))

    def run_ad():
        return elfi.AdaptiveDistanceSMC(m['d'], batch_size=10000, seed=5, device_proposal=dp,
                                        distributed=False, max_parallel_batches=2).sample(
            1000, rounds=3, quantile=0.3, bar=False)
    ad = run_ad()
    assert len(ad.populations) == 3
    assert np.all(np.isfinite(ad.samples_array)) and in_support(ad.samples)
    assert np.array_equal(ad.samples_array, run_ad().samples_array)
