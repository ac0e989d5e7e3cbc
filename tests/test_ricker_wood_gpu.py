"""Wood's 13 Ricker statistics on the device (elfi_b200/csrc/ricker_wood.cu):

* ops.wood_summaries against the host definition (ricker.wood_statistics) on device-simulated
  counts, to the contract of include/elfi_b200.h: columns 0..7 bit for bit, the cubic coefficients
  and the autoregression within their bounds, the rank rule's branch exactly, NaN rows;
* determinism: repeated calls and single-row calls give the same bits;
* the 'Wood' node of get_device_model(summary='wood'), and throughput-mode BSL on that model
  against a parity-mode run of the same configuration.
"""
import numpy as np
import pytest
import scipy.stats as ss

import ricker_wood_cases as rwc

pytestmark = pytest.mark.gpu
TRUTH = (3.8, 0.3, 10.0)


def _np(t):
    return t.cpu().numpy()


def _params(B, seed):
    """Half the rows at the truth, half at prior draws (extinctions, bursts, NaN rates)."""
    rs = np.random.RandomState(seed)
    P = np.column_stack([ss.expon.rvs(np.e, 2, size=B, random_state=rs),
                         ss.truncnorm.rvs(0, 5, size=B, random_state=rs), rs.uniform(0, 100, B)])
    P[:B // 2] = TRUTH
    return P


def _counts(n_obs, B, seed):
    from elfi_b200 import ops
    return ops.sim_ricker(_params(B, seed), n_obs, seed=seed, want_data=True,
                          want_summaries=False)[0]


def _observed(n_obs):
    from elfi_b200.examples import ricker
    return ricker.stochastic_ricker(*TRUTH, n_obs=n_obs, random_state=np.random.RandomState(n_obs))


def _degenerate(n_obs):
    rs = np.random.RandomState(n_obs)
    ones = (rs.uniform(size=n_obs) < 0.5).astype(float)
    ones[0] = 1.0
    sevens = 7.0 * (rs.uniform(size=n_obs) < 0.5)
    sevens[1] = 7.0
    nan, inf = ones.copy(), sevens.copy()
    nan[n_obs // 2], inf[-1] = np.nan, np.inf
    return np.array([np.zeros(n_obs), ones, sevens, nan, inf])


def _check(Y, obs):
    from elfi_b200 import ops
    from elfi_b200.examples import ricker
    P = ricker.wood_design(obs)
    got = _np(ops.wood_summaries(Y, P))
    y = _np(Y)
    rwc.check(got, ricker.wood_statistics(y, P), y, P, exact_sums=True)
    return got


@pytest.mark.parametrize('n_obs', [7, 8, 31, 50, 128, 129, 500, 2047, 2048])
def test_kernel_matches_host_definition(n_obs):
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    from elfi_b200.examples import ricker
    obs = _observed(n_obs)
    for B in (0, 1, 33):
        Y = _counts(n_obs, B, seed=B + n_obs)
        if B == 33:
            Y[-5:] = dev.to_device(_degenerate(n_obs))
        got = _check(Y, obs)
        assert got.shape == (B, 13)
        if B == 33:
            kinds = [rwc.rank_kind(r) for r in _np(Y)]
            assert {'none', 'one', 'full'} <= set(kinds) and np.isnan(got[-2:]).all()
    # strided rows: ldY > n
    Y = _counts(n_obs, 40, seed=3)
    wide = dev.empty((40, n_obs + 5))
    wide[:, :n_obs] = Y
    got = _check(wide[:, :n_obs], obs)
    np.testing.assert_array_equal(got, _np(ops.wood_summaries(Y, ricker.wood_design(obs))))


def test_large_batch_repeatable_and_row_independent():
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    from elfi_b200.examples import ricker
    obs = _observed(50)
    P = dev.to_device(ricker.wood_design(obs))
    Y = _counts(50, 100_000, seed=11)
    got = _check(Y, obs)
    again = _np(ops.wood_summaries(Y, P))
    np.testing.assert_array_equal(again, got)
    for i in (0, 1, 31, 32, 49_999, 50_000, 99_999):
        np.testing.assert_array_equal(_np(ops.wood_summaries(Y[i:i + 1], P))[0], got[i])
    assert np.isfinite(got).all(axis=1).mean() > 0.5


def test_device_model_node_equals_kernel_on_its_counts():
    from elfi_b200 import ops
    from elfi_b200.examples import ricker
    m, dp = ricker.get_device_model(seed_obs=2, summary='wood')
    out = m.generate(1000, ['Ricker', 'Wood'], seed=5)
    data = out['Ricker'].materialize()
    want = ops.wood_summaries(data, ricker.wood_design(m.observed['Ricker']))
    np.testing.assert_array_equal(_np(out['Wood']), _np(want))
    assert tuple(out['Wood'].shape) == (1000, 13)


# ---------------------------------------------------------------------------- BSL
SIGMA = np.diag([0.01, 0.004, 0.25])
N_ITER, BURN = 800, 200
# Calibration: this configuration run on an H100 in both modes (parity mode = the host model, same
# seed, same whitening) for seeds 1..5.  Parity-mode posterior means were t1 3.79 .. 3.92 (sd
# 0.11 .. 0.19), t3 9.48 .. 9.93 (sd 0.41 .. 0.64); the throughput-mode means differed from them by
# |0.026|, 0.112, 0.142, 0.045, 0.014 (t1) and |0.068|, 0.302, 0.443, 0.166, 0.007 (t3), Monte Carlo
# error of 600 correlated draws.  The tolerances are about three times the largest difference.
T1_TOL, T3_TOL = 0.4, 1.3


def _whitening():
    """A common scale for the statistics: their standard deviations at the truth (host model)."""
    from elfi_b200.examples import ricker
    m = ricker.get_model(n_obs=50, seed_obs=2, summary='wood')
    pilot = m.generate(2000, ['Wood'], with_values=dict(zip(['t1', 't2', 't3'], TRUTH)),
                       seed=1)['Wood']
    return np.diag(1 / np.std(pilot, axis=0))


def _bsl(throughput, seed, n_chains=1, n_iter=N_ITER, burn_in=BURN):
    from elfi_b200 import bsl
    from elfi_b200.examples import ricker
    lik = bsl.standard_likelihood(whitening=_whitening())
    if throughput:
        m, dp = ricker.get_device_model(n_obs=50, seed_obs=2, summary='wood')
    else:
        m, dp = ricker.get_model(n_obs=50, seed_obs=2, summary='wood'), None
    sampler = bsl.BSL(m, 500, ['Wood'], likelihood=lik, seed=seed, device_proposal=dp)
    params0 = np.tile(TRUTH, (n_chains, 1)) if n_chains > 1 else np.array(TRUTH)
    res = sampler.sample(n_iter, SIGMA, params0=params0, burn_in=burn_in, n_chains=n_chains)
    return sampler, res


def test_throughput_bsl_matches_parity_mode():
    _, par = _bsl(False, seed=1)
    sampler, thr = _bsl(True, seed=1)
    assert np.all(np.isfinite(sampler.state['logposterior']))
    assert 0 < thr.acc_rate < 1
    for name, tol in (('t1', T1_TOL), ('t3', T3_TOL)):
        a, b = np.mean(thr.samples[name]), np.mean(par.samples[name])
        assert abs(a - b) < tol, (name, a, b)


def test_lockstep_chains():
    sampler, res = _bsl(True, seed=3, n_chains=4, n_iter=200, burn_in=50)
    assert np.all(np.isfinite(sampler.state['logposterior']))
    assert res.chains.shape == (4, 200, 3)
    assert np.all((res.acc_rates > 0) & (res.acc_rates < 1))
