"""BSL's host logic under the CPU double of the C ABI: the host MA2 model reproduces the reference's
chains, penalty selection and whitening matrix (tests/golden/gen_golden_bsl.py)."""
import numpy as np
import pytest

import abi_double
import bsl_double
from elfi_b200 import bsl
from elfi_b200.examples import ma2

SIGMA = np.array([[.02, .01], [.01, .02]])


def _model():
    return ma2.get_model(n_obs=50, true_params=[.6, .2], seed_obs=4)


def _likelihood(name, g):
    if name == 'unbiased':
        return bsl.unbiased_likelihood()
    if name == 'whitened':
        return bsl.standard_likelihood(shrinkage='warton', penalty=g['penalty'], whitening=g['W'])
    return None


def run_chain(name, g):
    kw = dict(burn_in=50, logit_transform_bound=[[-2., 2.], [-1., 1.]]) if name == 'bounded' else {}
    sampler = bsl.BSL(_model(), 500, ['MA2'], likelihood=_likelihood(name, g), seed=123)
    res = sampler.sample(200, sigma_proposals=SIGMA, params0=np.array([.6, .2]), **kw)
    return sampler, res


def check_chain(name, g, sampler, res):
    chain = np.column_stack([res.samples_all[p] for p in ['t1', 't2']])
    np.testing.assert_array_equal(chain, g[name + '_samples_all'])
    lp, ref = sampler.state['logposterior'], g[name + '_logposterior']
    assert np.all(np.abs(lp - ref) <= 1e-9 * (1 + np.abs(ref)))
    assert res.acc_rate == float(g[name + '_acc_rate'])
    assert res.n_sim == int(g[name + '_n_sim'])
    burn = res.burn_in
    np.testing.assert_array_equal(res.samples['t1'], chain[burn:, 0])


@pytest.mark.parametrize('name', ['standard', 'unbiased', 'bounded', 'whitened'])
def test_chain_matches_reference(cpu_double, monkeypatch, golden, name):
    abi_double.install(monkeypatch, bsl_double.TABLE)
    g = golden('bsl_chains')
    sampler, res = run_chain(name, g)
    check_chain(name, g, sampler, res)
    assert cpu_double.CALLS.count('elfi_b200_synlik_f64') == res.n_sim // 500   # one per round
    ess = res.compute_ess()
    assert set(ess) == {'t1', 't2'} and all(v > 0 for v in ess.values())


def test_whitening_matrix_and_penalty(cpu_double, monkeypatch, golden):
    abi_double.install(monkeypatch, bsl_double.TABLE)
    g = golden('bsl_chains')
    W = bsl.estimate_whitening_matrix(_model(), 5000, np.array([.6, .2]), ['MA2'], seed=1)
    np.testing.assert_array_equal(W, g['W'])
    pen, std = bsl.select_penalty(_model(), 100, np.array([.6, .2]), ['MA2'], M=10,
                                  shrinkage='warton', whitening=g['W'], sigma=1.5, seed=1)
    np.testing.assert_array_equal(pen, g['penalty'])
    assert np.all(np.abs(std - g['penalty_std']) <= 1e-8)
    # all ten simulation sets and thirty penalties in one call
    assert cpu_double.CALLS.count('elfi_b200_synlik_f64') == 1


def test_params0_outside_support_and_host_callable(cpu_double, monkeypatch):
    abi_double.install(monkeypatch, bsl_double.TABLE)
    with pytest.raises(ValueError, match='outside prior support'):
        bsl.BSL(_model(), 100, ['MA2'], seed=1).sample(5, SIGMA, params0=[0.5, -0.9])
    seen = []

    def host_lik(ssx, ssy):
        seen.append((type(ssx), ssx.shape, ssy.shape))
        return bsl_double.synlik(ssx, ssy)

    res = bsl.BSL(_model(), 100, ['MA2'], likelihood=host_lik, seed=1).sample(
        5, SIGMA, params0=[.6, .2])
    assert res.n_sim == 100 * len(seen)
    assert all(t is np.ndarray and s == (100, 50) and o == (1, 50) for t, s, o in seen)
