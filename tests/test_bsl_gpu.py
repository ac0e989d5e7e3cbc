"""The device synthetic likelihood (elfi_b200_synlik_f64) against its NumPy restatement, its
failure and determinism rules, and BSL end to end on the host and device models."""
import numpy as np
import pytest
import torch

import bsl_double
from elfi_b200 import bsl, ops
from elfi_b200.examples import ma2, scratch_assay

pytestmark = pytest.mark.gpu

COND_MAX = 1e6
SIGMA = np.array([[.02, .01], [.01, .02]])


def groups(G, n, d, cond, rs):
    """(G, n, d) summaries whose sample covariances have condition number exactly `cond` (up to
    rounding): centred orthonormal columns, scaled, rotated and shifted."""
    out = np.empty((G, n, d))
    for g in range(G):
        q, _ = np.linalg.qr(np.column_stack([np.ones(n), rs.randn(n, d)]))
        rot, _ = np.linalg.qr(rs.randn(d, d))
        scales = np.sqrt(np.geomspace(1.0, cond, d)) * np.sqrt(n - 1)
        out[g] = (q[:, 1:] * scales) @ rot * rs.uniform(0.5, 2.0) + rs.randn(d)
    return out


def assert_conditioned(S, W=None):
    for X in S:
        sig = np.atleast_2d(np.cov(X, rowvar=False))
        if W is not None:
            sig = W @ sig @ W.T
        assert np.linalg.cond(sig) <= COND_MAX


def assert_close(dev_ll, ref):
    got = dev_ll.cpu().numpy()
    assert got.shape == ref.shape
    assert np.all(np.isfinite(ref))
    assert np.all(np.abs(got - ref) <= 1e-9 * (1 + np.abs(ref))), np.max(np.abs(got - ref))


def observed(S, rs):
    return S[0].mean(axis=0) + rs.randn(S.shape[2]) * S[0].std(axis=0)


CASES = [(d, n) for d in (1, 2, 31, 32, 33, 64, 145, 160)
         for n in sorted({d + 1, max(d + 8, 300), 5000 if d in (1, 33, 145, 160) else d + 1})]


@pytest.mark.parametrize('d,n', CASES)
def test_standard_and_unbiased_match_oracle(d, n):
    rs = np.random.RandomState(d * 7919 + n)
    G = 3
    S = groups(G, n, d, 1e4, rs)
    assert_conditioned(S)
    y = observed(S, rs)
    assert_close(ops.synlik(S, y), bsl_double.synlik(S, y))
    if n > d + 3:
        assert_close(ops.synlik(S, y, estimator='unbiased'), bsl_double.synlik(S, y, 'unbiased'))


@pytest.mark.parametrize('d,n', [(2, 50), (33, 300), (145, 1000), (160, 5000)])
def test_warton_and_whitening_match_oracle(d, n):
    rs = np.random.RandomState(d + n)
    S = groups(4, n, d, 1e3, rs)
    y = observed(S, rs)
    pens = np.linspace(0.0, 1.0, 30)
    assert_close(ops.synlik(S, y, penalties=pens), bsl_double.synlik(S, y, penalties=pens))
    W = np.eye(d) + 0.1 * rs.randn(d, d) / np.sqrt(d)
    assert_conditioned(S, W)
    assert_close(ops.synlik(S, y, whitening=W), bsl_double.synlik(S, y, W=W))
    assert_close(ops.synlik(S, y, penalties=pens[:7], whitening=W),
                 bsl_double.synlik(S, y, penalties=pens[:7], W=W))


def test_strided_rows_and_gapped_groups():
    rs = np.random.RandomState(5)
    d, n, G = 31, 120, 600
    S = groups(G, n, d, 1e4, rs)
    y = observed(S, rs)
    ref = bsl_double.synlik(S, y, penalties=[0.0, 0.3])
    # rows of d + 5 values, every other group
    big = torch.zeros((2 * G, n, d + 5), dtype=torch.float64, device='cuda')
    view = big[::2, :, 2:2 + d]
    view.copy_(torch.from_numpy(S))
    assert view.stride() == (2 * n * (d + 5), d + 5, 1)
    assert_close(ops.synlik(view, y, penalties=[0.0, 0.3]), ref)
    # groups interleaved row by row: a (n, G, d) array read as (G, n, d)
    inter = torch.from_numpy(np.ascontiguousarray(S.transpose(1, 0, 2))).cuda().transpose(0, 1)
    assert_close(ops.synlik(inter, y, penalties=[0.0, 0.3]), ref)


def test_failures_stay_in_their_group():
    rs = np.random.RandomState(11)
    d, n = 12, 200
    S = groups(6, n, d, 1e3, rs)
    y = observed(S, rs)
    S[1, 17, 3] = np.nan
    S[2, 0, 0] = np.inf
    S[3, :, 5] = S[3, :, 2]            # duplicated column
    S[4, :, 7] = 2.5                   # constant column
    ll = ops.synlik(S, y).cpu().numpy()
    assert np.all(np.isneginf(ll[1:5]))
    assert np.all(np.isfinite(ll[[0, 5]]))
    assert np.array_equal(ll[[0, 5]], ops.synlik(S[[0, 5]], y).cpu().numpy())
    assert np.all(np.isneginf(bsl_double.synlik(S, y)[1:5]))
    llk = ops.synlik(S, y, penalties=[0.2, 0.9]).cpu().numpy()
    assert np.all(np.isneginf(llk[1:3])) and np.all(np.isfinite(llk[[0, 5]]))


def test_deterministic_and_independent_of_batching():
    rs = np.random.RandomState(3)
    d, n, G = 145, 1000, 20        # 20 groups walk their row chunks in one CTA; one group splits
    S = groups(G, n, d, 1e4, rs)
    y = observed(S, rs)
    pens = [0.0, 0.25, 0.5]
    first = ops.synlik(S, y, penalties=pens).cpu().numpy()
    for _ in range(3):
        assert np.array_equal(ops.synlik(S, y, penalties=pens).cpu().numpy(), first)
    for g in (0, 7, 19):
        assert np.array_equal(ops.synlik(S[g], y, penalties=pens).cpu().numpy()[0], first[g])
        for k, p in enumerate(pens):
            assert ops.synlik(S[g], y, penalties=[p]).cpu().numpy()[0, 0] == first[g, k]
    assert np.array_equal(ops.synlik(S, y).cpu().numpy(), first[:, 0])


def _chain_model():
    return ma2.get_model(n_obs=50, true_params=[.6, .2], seed_obs=4)


@pytest.mark.parametrize('name', ['standard', 'unbiased', 'bounded', 'whitened'])
def test_golden_chains(golden, name):
    g = golden('bsl_chains')
    lik = {'unbiased': bsl.unbiased_likelihood(),
           'whitened': bsl.standard_likelihood(shrinkage='warton', penalty=g['penalty'],
                                               whitening=g['W'])}.get(name)
    kw = dict(burn_in=50, logit_transform_bound=[[-2., 2.], [-1., 1.]]) if name == 'bounded' else {}
    sampler = bsl.BSL(_chain_model(), 500, ['MA2'], likelihood=lik, seed=123)
    res = sampler.sample(200, sigma_proposals=SIGMA, params0=np.array([.6, .2]), **kw)
    chain = np.column_stack([res.samples_all[p] for p in ['t1', 't2']])
    np.testing.assert_array_equal(chain, g[name + '_samples_all'])
    ref = g[name + '_logposterior']
    assert np.all(np.abs(sampler.state['logposterior'] - ref) <= 1e-9 * (1 + np.abs(ref)))
    assert res.acc_rate == float(g[name + '_acc_rate'])
    assert res.n_sim == int(g[name + '_n_sim'])


def test_golden_penalty_selection(golden):
    g = golden('bsl_chains')
    pen, std = bsl.select_penalty(_chain_model(), 100, np.array([.6, .2]), ['MA2'], M=10,
                                  shrinkage='warton', whitening=g['W'], sigma=1.5, seed=1)
    np.testing.assert_array_equal(pen, g['penalty'])
    assert np.all(np.abs(std - g['penalty_std']) <= 1e-8)


@pytest.mark.parametrize('likelihood', [None, bsl.unbiased_likelihood()])
def test_device_ma2_posterior(likelihood):
    m = ma2.get_device_model(n_obs=50, seed_obs=4)
    res = bsl.BSL(m, 500, ['MA2'], likelihood=likelihood, seed=123).sample(
        2000, sigma_proposals=SIGMA, params0=np.array([.6, .2]))
    means = [np.mean(res.samples['t1']), np.mean(res.samples['t2'])]
    assert abs(means[0] - .6) < .15 and abs(means[1] - .2) < .15, means
    assert 0 < res.acc_rate < 1


def test_device_scratch_assay_runs():
    m, _ = scratch_assay.get_device_model(seed_obs=7)
    sampler = bsl.BSL(m, 500, seed=5)
    assert sampler.observed.size == 145
    res = sampler.sample(40, sigma_proposals=np.diag([4e-4, 1e-7]),
                         params0=np.array([0.25, 0.002]))
    lp = sampler.state['logposterior']
    assert np.isfinite(lp[0])
    for p in ('pm', 'pp'):
        assert np.all((res.samples_all[p] > 0) & (res.samples_all[p] < 1))
    assert 0 < res.acc_rate < 1
