"""Lock-step BSL chains under the CPU double of the C ABI: parity mode on the host MA2 model equals
C reference-style chains sharing one batch stream (tests/bsl_chains_double.py), and throughput
mode's host logic runs end to end with the NumPy restatement of elfi_b200_bsl_mh_step_f64."""
import numpy as np
import pytest

import abi_double
import bsl_chains_double
import bsl_double
import priors_double
from elfi_b200 import bsl
from elfi_b200.examples import ma2

BOUNDS = [[-2., 2.], [-1., 1.]]
SIGMA_WIDE = np.diag([4.0, 4.0])            # in the logit space: about half the proposals leave
PARAMS0 = np.array([[.6, .2], [.3, .1], [-.2, -.3]])


def _model():
    return ma2.get_model(n_obs=50, true_params=[.6, .2], seed_obs=4)


def _record_groups(monkeypatch):
    groups = []

    def synlik_f64(*args):
        groups.append(args[4])
        return bsl_double.synlik_f64(*args)
    monkeypatch.setitem(bsl_double.TABLE, 'elfi_b200_synlik_f64', synlik_f64)
    return groups


def test_parity_chains_match_restatement(cpu_double, monkeypatch):
    groups = _record_groups(monkeypatch)
    abi_double.install(monkeypatch, bsl_double.TABLE)
    n, n_round, b, seed = 40, 100, 50, 17
    sampler = bsl.BSL(_model(), n_round, ['MA2'], batch_size=b, seed=seed)
    res = sampler.sample(n, SIGMA_WIDE, params0=PARAMS0, burn_in=5, logit_transform_bound=BOUNDS,
                         n_chains=3)
    chains, lp, acc, n_batches = bsl_chains_double.parity_chains(
        _model(), 'MA2', n_round, b, seed, n, SIGMA_WIDE, PARAMS0, burn_in=5, bounds=BOUNDS)
    np.testing.assert_array_equal(res.chains, chains)
    got = sampler.state['logposterior']
    assert got.shape == (3, n)
    assert np.all(np.abs(got - lp) <= 1e-9 * (1 + np.abs(lp)))
    # some proposals left the support, and some iterations had no chain inside it
    assert np.any(chains[:, 1:] == chains[:, :-1])
    simulated = n_batches // (n_round // b)
    assert simulated < n
    # an all-outside iteration consumes no batch; n_sim counts every simulated row
    assert res.n_sim == n_batches * 3 * b == sampler.state['n_batches'] * 3 * b
    assert groups == [3] * simulated            # one likelihood call per simulated iteration
    np.testing.assert_array_equal(res.acc_rates, acc / (n - 5))
    assert res.acc_rate == acc.sum() / (3 * (n - 5))
    assert res.n_chains == 3 and res.samples_all['t1'].shape == (3, n)
    np.testing.assert_array_equal(res.samples['t2'], chains[:, 5:, 1].reshape(-1))
    ess = res.compute_ess()
    assert set(ess) == {'t1', 't2'} and all(v > 0 for v in ess.values())


def test_parity_chains_without_bounds_and_prior_start(cpu_double, monkeypatch):
    abi_double.install(monkeypatch, bsl_double.TABLE)
    sigma = np.array([[.02, .01], [.01, .02]])
    sampler = bsl.BSL(_model(), 100, ['MA2'], seed=3)
    res = sampler.sample(12, sigma, n_chains=4)
    start = sampler.model.generate(4, ['t1', 't2'], seed=3)
    params0 = np.column_stack([start['t1'], start['t2']])
    np.testing.assert_array_equal(res.chains[:, 0], params0)
    chains, lp, _, n_batches = bsl_chains_double.parity_chains(_model(), 'MA2', 100, 100, 3, 12,
                                                              sigma, params0)
    np.testing.assert_array_equal(res.chains, chains)
    assert np.all(np.abs(sampler.state['logposterior'] - lp) <= 1e-9 * (1 + np.abs(lp)))
    assert res.n_sim == n_batches * 4 * 100


def test_one_chain_is_the_single_chain_sampler(cpu_double, monkeypatch):
    """n_chains=1 is the same code path: the restatement with C = 1 is the reference's chain."""
    abi_double.install(monkeypatch, bsl_double.TABLE)
    sampler = bsl.BSL(_model(), 100, ['MA2'], batch_size=50, seed=9)
    res = sampler.sample(15, SIGMA_WIDE, params0=[.6, .2], logit_transform_bound=BOUNDS)
    chains, lp, acc, n_batches = bsl_chains_double.parity_chains(
        _model(), 'MA2', 100, 50, 9, 15, SIGMA_WIDE, PARAMS0[:1], bounds=BOUNDS)
    np.testing.assert_array_equal(np.column_stack([res.samples_all['t1'], res.samples_all['t2']]),
                                  chains[0])
    assert sampler.state['logposterior'].shape == (15,)
    assert res.acc_rate == acc[0] / 15 and res.n_sim == n_batches * 50
    assert 'chains' not in res.meta


def test_argument_errors(cpu_double, monkeypatch):
    abi_double.install(monkeypatch, bsl_double.TABLE)
    sigma = np.array([[.02, .01], [.01, .02]])
    with pytest.raises(ValueError, match=r'params0 must be \(2,\) or \(3, 2\)'):
        bsl.BSL(_model(), 100, ['MA2'], seed=1).sample(5, sigma, params0=np.zeros((2, 2)),
                                                      n_chains=3)
    with pytest.raises(ValueError, match=r'outside prior support \(chain 1\)'):
        bsl.BSL(_model(), 100, ['MA2'], seed=1).sample(
            5, sigma, params0=[[.6, .2], [.5, -.9], [.1, .1]], n_chains=3)
    with pytest.raises(ValueError, match='n_chains'):
        bsl.BSL(_model(), 100, ['MA2'], seed=1).sample(5, sigma, n_chains=0)
    with pytest.raises(ValueError, match='device likelihood'):
        m, dp = ma2.get_uniform_device_model(n_obs=10, seed_obs=4)
        bsl.BSL(m, 100, ['MA2'], likelihood=bsl_double.synlik, device_proposal=dp)


def test_throughput_mode_host_logic(cpu_double, monkeypatch):
    abi_double.install(monkeypatch, bsl_double.TABLE, priors_double.TABLE, bsl_chains_double.TABLE)
    m, dp = ma2.get_uniform_device_model(n_obs=20, seed_obs=4)
    sigma = np.diag([.05, .05])

    def run():
        del cpu_double.CALLS[:]
        s = bsl.BSL(m, 60, ['MA2'], batch_size=30, seed=11, device_proposal=dp)
        return s, s.sample(25, sigma, params0=[.6, .2], burn_in=5, n_chains=4,
                           logit_transform_bound=BOUNDS)
    sampler, res = run()
    calls = list(cpu_double.CALLS)
    assert calls.count('elfi_b200_bsl_mh_step_f64') == 25
    assert calls.count('elfi_b200_synlik_f64') == 25
    # every iteration simulates: two batches of 4 x 30 rows
    assert res.n_sim == 25 * 2 * 4 * 30 and sampler.state['n_batches'] == 50
    assert res.chains.shape == (4, 25, 2)
    np.testing.assert_array_equal(res.chains[:, 0], np.tile([.6, .2], (4, 1)))
    lp = sampler.state['logposterior']
    assert lp.shape == (4, 25) and np.all(np.isfinite(lp))
    assert np.all((np.abs(res.chains[..., 0]) <= 2) & (np.abs(res.chains[..., 1]) <= 1))
    assert 0 < res.acc_rate < 1 and res.acc_rates.shape == (4,)
    # a rejected step repeats the state and its log posterior
    same = np.all(res.chains[:, 1:] == res.chains[:, :-1], axis=2)
    np.testing.assert_array_equal(lp[:, 1:][same], lp[:, :-1][same])
    _, again = run()
    np.testing.assert_array_equal(again.chains, res.chains)
