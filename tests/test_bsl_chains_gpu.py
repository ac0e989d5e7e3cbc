"""Lock-step BSL chains on the device: parity mode against its NumPy restatement, the device
Metropolis-Hastings step (elfi_b200_bsl_mh_step_f64) against its NumPy replay, and throughput mode
end to end on the MA2 and scratch assay device models."""
import numpy as np
import pytest
import torch

import bsl_chains_double as bcd
import elfi_b200 as elfi
from elfi_b200 import bsl, mcmc, ops
from elfi_b200.examples import ma2, mg1, scratch_assay

pytestmark = pytest.mark.gpu

BOUNDS = [[-2., 2.], [-1., 1.]]
SIGMA_WIDE = np.diag([4.0, 4.0])
PARAMS0 = np.array([[.6, .2], [.3, .1], [-.2, -.3]])


def test_parity_mode_matches_restatement():
    m = ma2.get_model(n_obs=50, true_params=[.6, .2], seed_obs=4)
    sampler = bsl.BSL(m, 100, ['MA2'], batch_size=50, seed=17)
    res = sampler.sample(40, SIGMA_WIDE, params0=PARAMS0, burn_in=5, logit_transform_bound=BOUNDS,
                         n_chains=3)
    chains, lp, acc, n_batches = bcd.parity_chains(
        ma2.get_model(n_obs=50, true_params=[.6, .2], seed_obs=4), 'MA2', 100, 50, 17, 40,
        SIGMA_WIDE, PARAMS0, burn_in=5, bounds=BOUNDS)
    np.testing.assert_array_equal(res.chains, chains)
    got = sampler.state['logposterior']
    assert np.all(np.abs(got - lp) <= 1e-9 * (1 + np.abs(lp)))
    np.testing.assert_array_equal(res.acc_rates * 35, acc)
    assert res.n_sim == n_batches * 3 * 50


def _uniform_table(p, rs):
    lo = rs.uniform(-1.5, -0.5, p)
    return np.array([[0, lo[a], rs.uniform(1.5, 3.0), 0, 0] for a in range(p)]), None


def _case(p, kind, rs):
    if kind == 'mg1':
        dp = elfi.DeviceModelPrior(mg1.get_model(seed_obs=1), conditional=True)
        x0 = np.array([2.0, 6.0, 0.2])
        return dp.specs, dp.sources, x0, np.diag([1.0, 4.0, 0.02])
    specs, sources = _uniform_table(p, rs)
    x0 = specs[:, 1] + 0.5 * specs[:, 2]
    a = rs.randn(p, p) * 0.2
    return specs, sources, x0, (a @ a.T + np.eye(p) * 0.5) * min(1.0, 4.0 / p)


@pytest.mark.parametrize('p,kind', [(1, 'plain'), (2, 'plain'), (3, 'plain'), (16, 'plain'),
                                    (1, 'bounds'), (2, 'bounds'), (3, 'bounds'), (16, 'bounds'),
                                    (3, 'mg1')])
def test_mh_step_matches_replay(p, kind):
    rs = np.random.RandomState(100 * p + len(kind))
    specs, sources, x0, cov = _case(p, kind, rs)
    bounds = None
    if kind == 'bounds':
        # wider than the supports, one side infinite for some parameters: proposals still leave
        bounds = np.column_stack([specs[:, 1] - 1.0, specs[:, 1] + specs[:, 2] + 1.0])
        bounds[::3, 0] = -np.inf
        bounds[1::3, 1] = np.inf
    tables = ops.bsl_mh_tables(specs, cov, sources, bounds)
    C, n, b, seed, burn = 300, 12, 5, 987654321, 3
    dev = dict(prop=torch.tensor(np.tile(x0, (C, 1)) + 0.01 * rs.randn(C, p), device='cuda'),
               chains=torch.zeros((C, n, p), dtype=torch.float64, device='cuda'),
               logpost=torch.zeros((C, n), dtype=torch.float64, device='cuda'),
               n_acc=torch.zeros(C, dtype=torch.int64, device='cuda'))
    dev['prop_lp'] = ops.prior_logpdf(dev['prop'], specs, sources)
    rows = torch.zeros((p, C * b), dtype=torch.float64, device='cuda')
    outside = decided = 0
    for t in range(n):
        ll = torch.tensor(rs.randn(C) * 3.0 - 50.0, device='cuda')
        host = {k: v.cpu().numpy().copy() for k, v in dev.items()}
        r, accept, margin = bcd.mh_step(t, tables[0], tables[1], tables[2], seed, burn,
                                        ll.cpu().numpy(), host['prop'], host['prop_lp'],
                                        host['chains'], host['logpost'], host['n_acc'])
        ops.bsl_mh_step(tables, t, ll, dev['prop'], dev['prop_lp'], dev['chains'],
                        dev['logpost'], dev['n_acc'], rows, seed, burn)
        got = {k: v.cpu().numpy() for k, v in dev.items()}
        sure = margin >= 1e-12
        decided += int(np.sum(np.isfinite(margin)))
        # logposteriors exact given the inputs, states and counters equal where the decision is sure
        np.testing.assert_array_equal(got['logpost'][sure, t], host['logpost'][sure, t])
        np.testing.assert_array_equal(got['chains'][sure, t], host['chains'][sure, t])
        if t + 1 < n:
            # the next proposals, their log priors and the next batch's rows
            ok = sure
            ref = host['prop'][ok]
            assert np.all(np.abs(got['prop'][ok] - ref) <= 1e-13 * (1 + np.abs(ref)))
            lp_ref = host['prop_lp'][ok]
            fin = np.isfinite(lp_ref)
            np.testing.assert_array_equal(np.isfinite(got['prop_lp'][ok]), fin)
            assert np.all(np.abs(got['prop_lp'][ok][fin] - lp_ref[fin])
                          <= 1e-12 * (1 + np.abs(lp_ref[fin])))
            outside += int(np.sum(~fin))
            rr = rows.cpu().numpy().T.reshape(C, b, p)
            assert np.all(rr == rr[:, :1])
            assert np.all(np.abs(rr[ok, 0] - r[ok]) <= 1e-13 * (1 + np.abs(r[ok])))
        # the replay of the next step starts from the device's state, so the two never drift apart
    assert outside > 0 and decided > 0
    # the counters: accepted steps from burn_in on
    moved = np.any(got['chains'][:, burn:] != got['chains'][:, burn - 1:-1], axis=2).sum(axis=1)
    assert np.all(got['n_acc'] >= moved)


def test_mh_step_is_deterministic_and_independent_of_c():
    specs, _ = _uniform_table(2, np.random.RandomState(1))
    tables = ops.bsl_mh_tables(specs, np.eye(2) * 0.3)

    def run(C):
        prop = torch.tensor(np.tile(specs[:, 1] + 0.5 * specs[:, 2], (C, 1)), device='cuda')
        lp = ops.prior_logpdf(prop, specs)
        chains = torch.zeros((C, 6, 2), dtype=torch.float64, device='cuda')
        logpost = torch.zeros((C, 6), dtype=torch.float64, device='cuda')
        n_acc = torch.zeros(C, dtype=torch.int64, device='cuda')
        rows = torch.zeros((2, C * 3), dtype=torch.float64, device='cuda')
        for t in range(6):
            ll = torch.full((C,), -10.0 - t, dtype=torch.float64, device='cuda')
            ops.bsl_mh_step(tables, t, ll, prop, lp, chains, logpost, n_acc, rows, 5)
        return chains.cpu().numpy(), logpost.cpu().numpy()
    a, la = run(40)
    b, lb = run(40)
    c, lc = run(7)
    np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(la, lb)
    np.testing.assert_array_equal(a[:7], c)
    np.testing.assert_array_equal(la[:7], lc)


def _ma2_throughput(seed):
    m, dp = ma2.get_uniform_device_model(n_obs=50, seed_obs=4)
    rs = np.random.RandomState(0)
    params0 = np.column_stack([rs.uniform(.3, .9, 64), rs.uniform(0., .4, 64)])
    sampler = bsl.BSL(m, 500, ['MA2'], seed=seed, device_proposal=dp)
    res = sampler.sample(600, np.array([[.06, .03], [.03, .06]]), params0=params0, burn_in=100,
                         n_chains=64)
    return sampler, res


def test_throughput_mode_ma2_posterior():
    sampler, res = _ma2_throughput(123)
    means = [np.mean(res.samples['t1']), np.mean(res.samples['t2'])]
    assert abs(means[0] - .6) < .1 and abs(means[1] - .2) < .1, means
    for i in range(2):
        assert mcmc.gelman_rubin_statistic(res.chains[:, 100:, i]) < 1.1
    assert 0 < res.acc_rate < 1
    assert np.all(np.isfinite(sampler.state['logposterior']))
    assert res.n_sim == 600 * 64 * 500
    _, again = _ma2_throughput(123)
    np.testing.assert_array_equal(again.chains, res.chains)
    np.testing.assert_array_equal(again.acc_rates, res.acc_rates)


@pytest.mark.parametrize('throughput', [False, True])
def test_scratch_assay_chains_run(throughput):
    m, dp = scratch_assay.get_device_model(seed_obs=7)
    sampler = bsl.BSL(m, 300, seed=5, device_proposal=dp if throughput else None)
    assert sampler.observed.size == 145
    res = sampler.sample(30, np.diag([4e-4, 1e-7]), params0=np.array([0.25, 0.002]),
                         n_chains=16)
    assert np.all(np.isfinite(sampler.state['logposterior']))
    assert res.chains.shape == (16, 30, 2)
    assert np.all((res.chains > 0) & (res.chains < 1))
