"""Stock scipy.stats priors on the device (elfi_b200/csrc/prior.cu, the support-3 and p <= 16
proposals of simulate.cu, elfi_b200.DeviceModelPrior).

Kernel level: every prior draw and proposal is compared element by element with the NumPy replay
of its Philox stream (tests/prior_replay.py) at ulp-level tolerances derived from the operations;
rows whose Marsaglia-Tsang or support decision lies within 1e-9 of its bound could go either way
in the last bits and are excluded (at most max(2, 1e-4 B) of them).  The log densities are
compared with scipy through ModelPrior.  Sampler level: a six-parameter model with one prior of
every kind runs Rejection and SMC with device priors and proposals against the host path, and the
g-and-k model with stock priors runs AdaptiveDistanceSMC against its bespoke device proposal.
"""
from functools import partial

import numpy as np
import pytest
import scipy.stats as ss

import device_prior_cases as cases
import prior_replay as pr

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -52


def _np(t):
    return t.cpu().numpy()


def _spec(kind, params):
    from elfi_b200.priors import prior_spec
    return np.asarray(prior_spec(kind, params), dtype=np.float64)


def _within(got, want, tol, what):
    bad = ~(np.abs(got - want) <= tol)
    assert not bad.any(), '{}: {} of {} differ, first at {}: {} vs {} (tol {})'.format(
        what, int(bad.sum()), bad.size, np.argwhere(bad)[0], got[bad][0], want[bad][0],
        np.broadcast_to(tol, bad.shape)[bad][0])


# ------------------------------------------------------------------------------ prior_rvs
SHAPES = [(1, 3, 0), (255, 3, 0), (257, 3, 7), (100000, 2 ** 32 + 5, 2 ** 32 - 50000)]


@pytest.mark.parametrize('B,seed,offset', SHAPES)
@pytest.mark.parametrize('case', cases.KIND_CASES, ids=cases.case_id)
def test_prior_rvs_matches_replay(case, B, seed, offset):
    from elfi_b200 import ops
    spec = _spec(*case)
    x = _np(ops.prior_rvs(spec, B, seed=seed, offset=offset))
    xr, err, trial, margin = pr.prior_rvs(spec, B, seed, offset)
    amb = margin < 1e-9
    assert amb.sum() <= max(2, 1e-4 * B), int(amb.sum())
    _within(x[~amb], xr[~amb], err[~amb], str(case))
    lo, hi = pr.support(spec)
    assert np.all((x >= lo) & (x <= hi))
    if case[0] in ('gamma', 'beta') and B >= 100000:
        assert (trial[~amb] >= 1).sum() > 0           # the trial loop is exercised ...
        assert trial.max() < pr.MAX_TRIALS - 1          # ... and far from its bound


@pytest.mark.parametrize('case', cases.KIND_CASES, ids=cases.case_id)
def test_prior_rvs_sharding_invariant_and_follows_scipy(case):
    """Two offset halves equal one call bit for bit; 1e6 draws pass KS against scipy."""
    from elfi_b200 import ops
    spec = _spec(*case)
    B, seed = 1000000, 2 ** 33 + 9
    x = _np(ops.prior_rvs(spec, B, seed=seed))
    h1 = _np(ops.prior_rvs(spec, 400001, seed=seed))
    h2 = _np(ops.prior_rvs(spec, B - 400001, seed=seed, offset=400001))
    assert np.array_equal(np.concatenate([h1, h2]), x)
    assert ss.kstest(x, cases.frozen(*case).cdf).pvalue > 1e-3
    assert np.unique(x).size > 0.99 * B


def test_prior_rvs_refuses_bad_parameters():
    from elfi_b200 import _lib, ops
    with pytest.raises(ValueError, match='prior parameter 0: beta needs'):
        ops.prior_rvs([5, 0, 1, 0, 1], 10, seed=1)
    # the library checks too, and names the parameter
    from elfi_b200 import device as dev
    bad = np.array([2.0, 3.0, 3.0, 0.0, 1.0])
    out = dev.empty((4,))
    with pytest.raises(_lib.ElfiB200Error, match='prior parameter 0: truncnorm needs a < b'):
        _lib.call('elfi_b200_prior_rvs_f64', dev.context(), dev.ptr(bad), 4, 1, 0, dev.ptr(out),
                  dev.stream_ptr())
    table = np.array([[0.0, 0.0, 1.0, 0.0, 0.0], [4.0, -1.0, 0.0, 1.0, 0.0]])
    x = dev.zeros((3, 2))
    with pytest.raises(_lib.ElfiB200Error, match='prior parameter 1: gamma needs'):
        _lib.call('elfi_b200_prior_logpdf_f64', dev.context(), dev.ptr(x), 2, 3, 2, dev.ptr(table),
                  dev.ptr(out), dev.stream_ptr())


# ------------------------------------------------------------------------------ prior_logpdf
def _prior_model(priors):
    from elfi_b200 import model as em
    m = em.new_model()
    for i, (kind, params) in enumerate(priors):
        em.Prior(kind, *params, model=m, name='p{:02d}'.format(i))
    return m


@pytest.mark.parametrize('group', [cases.KIND_CASES[:16], cases.KIND_CASES[2:], cases.SIX_PRIORS,
                                   cases.KIND_CASES[5:6]], ids=['first16', 'last16', 'six', 'tail'])
def test_prior_logpdf_matches_model_prior(group):
    """ops.prior_logpdf against ModelPrior(model).logpdf (scipy through the graph) at points
    inside, outside, on the support edges and one ulp beyond: rtol 1e-13, exact infinities."""
    import elfi_b200 as elfi
    from elfi_b200 import ops
    m = _prior_model(group)
    dp = elfi.DeviceModelPrior(m)
    rs = np.random.RandomState(len(group))
    cols = []
    for kind, params in group:
        spec = _spec(kind, params)
        lo, hi = pr.support(spec)
        inside = cases.frozen(kind, params).rvs(size=3000, random_state=rs)
        flo = lo if np.isfinite(lo) else inside.min()
        fhi = hi if np.isfinite(hi) else inside.max()
        around = rs.uniform(flo - 0.2 * (fhi - flo), fhi + 0.2 * (fhi - flo), 1000)
        edges = [e for e in (lo, hi) if np.isfinite(e)]
        edge = np.array([f(e) for e in edges for f in (lambda v: v, lambda v: np.nextafter(v, np.inf),
                                                        lambda v: np.nextafter(v, -np.inf))] or [0.0])
        cols.append(np.concatenate([inside, around, np.resize(edge, 60)]))
    x = np.column_stack(cols)
    # rows with one coordinate on an edge and the rest inside
    for a, col in enumerate(cols):
        x[3000 + a::len(cols)][:20, a] = col[-60:-40]
    with np.errstate(all='ignore'):
        ref = elfi.ModelPrior(m).logpdf(x)
    got = _np(ops.prior_logpdf(x, dp.specs))
    assert np.array_equal(np.isposinf(got), np.isposinf(ref))
    assert np.array_equal(np.isneginf(got), np.isneginf(ref))
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    fin = np.isfinite(ref)
    assert fin.sum() > 1000
    np.testing.assert_allclose(got[fin], ref[fin], rtol=1e-13, atol=1e-13)
    # a row-strided view is read in place
    import torch
    store = torch.zeros((x.shape[0], x.shape[1] + 3), dtype=torch.float64, device='cuda')
    store[:, :x.shape[1]] = torch.from_numpy(x).cuda()
    assert np.array_equal(_np(ops.prior_logpdf(store[:, :x.shape[1]], dp.specs)), got, equal_nan=True)


# ------------------------------------------------------------------------------ gm_rvs
GM_KINDS = [('beta', (2.0, 3.0)), ('uniform', (-1.0, 2.0)), ('truncnorm', (0.0, 3.0)),
            ('gamma', (2.0, 0.0, 0.5)), ('expon', (0.0, 1.0)), ('norm', (0.0, 1.0)),
            ('gamma', (0.3,)), ('beta', (0.5, 0.5))]


def _gm_case(p, rs):
    priors = [GM_KINDS[a % len(GM_KINDS)] for a in range(p)]
    specs = np.array([_spec(*c) for c in priors])
    N = 700
    means = np.column_stack([cases.frozen(*c).rvs(size=N, random_state=rs) for c in priors])
    a = rs.randn(p, p)
    cov = (0.05 if p <= 5 else 0.02) * (a @ a.T / p + 0.5 * np.eye(p))
    w = rs.rand(N) ** 4
    w[0] = w[-1] = 0.0
    return specs, means, cov, w


@pytest.mark.parametrize('support', [0, 3])
@pytest.mark.parametrize('p', [1, 4, 5, 8, 16])
def test_gm_rvs_matches_replay(p, support):
    """Proposals for p <= 16 and support 3 vs the replay (means as a row-strided view, the
    device's own CDF table); support 3: every draw has a finite prior log density and the redraw
    path is exercised (> 5 % of the rows need a second trial)."""
    import torch
    from elfi_b200 import ops
    rs = np.random.RandomState(p * 10 + support)
    specs, means, cov, w = _gm_case(p, rs)
    N, B = means.shape[0], 20000
    store = torch.zeros((N, p + 3), dtype=torch.float64, device='cuda')
    store[:, :p] = torch.from_numpy(means).cuda()
    cdf = ops.gm_cdf(w, N)
    seed, offset = 2 ** 32 + 9, 2 ** 32 - 7
    x = _np(ops.gm_rvs(store[:, :p], cov, None, B, seed=seed, offset=offset, support=support,
                       cdf=cdf, prior=specs if support == 3 else None))
    L = np.linalg.cholesky(cov)
    xr, trial, comp, err, margin = pr.gm_rvs(means, L, _np(cdf), B, seed, offset, support,
                                             specs=specs)
    amb = margin < 1e-9
    assert amb.sum() <= max(2, 1e-4 * B), int(amb.sum())
    _within(x[~amb], xr[~amb], err[~amb, None], 'draws')
    assert np.all(w[comp] > 0) and np.all(trial >= 0)
    if support == 3:
        assert np.isfinite(pr.joint_logpdf(specs, x)).all()
        assert np.sum(trial >= 1) > 0.05 * B, np.mean(trial >= 1)
    if p <= 4 and support == 0:
        # the p <= 4 kernel and its replay are unchanged: the same particles
        x4 = _np(ops.gm_rvs(store[:, :p], cov, None, B, seed=seed, offset=offset, cdf=cdf))
        assert np.array_equal(x4, x)


def test_gm_rvs_support3_equals_box_for_uniform_priors():
    """With uniform priors, support 3 and the box support 2 accept the same region: the same
    particles (the wide kernel uses the p <= 4 kernel's blocks)."""
    from elfi_b200 import ops
    rs = np.random.RandomState(5)
    means = rs.uniform(0, 10, (300, 4))
    cov = np.eye(4) * 2.0
    specs = np.array([_spec('uniform', (0.0, 10.0))] * 4)
    w = rs.rand(300)
    b = _np(ops.gm_rvs(means, cov, w, 50000, seed=11, support=2, box=([0.0] * 4, [10.0] * 4)))
    c = _np(ops.gm_rvs(means, cov, w, 50000, seed=11, support=3, prior=specs))
    assert np.array_equal(b, c)
    assert np.all((c >= 0) & (c <= 10))


# ------------------------------------------------------------------------------ samplers
def _posterior_check(res, ref, what):
    """Posterior means within 4 Monte-Carlo standard errors of each other (ESS-based)."""
    a, b = res.sample_means_array, ref.sample_means_array
    se = []
    for r in (res, ref):
        w = r.weights if r.weights is not None else np.ones(r.n_samples)
        ess = w.sum() ** 2 / (w ** 2).sum()
        se.append(r.samples_array.std(axis=0) / np.sqrt(ess))
    tol = 4 * np.sqrt(se[0] ** 2 + se[1] ** 2)
    assert np.all(np.abs(a - b) <= tol), (what, a, b, tol)


def test_rejection_round0_draws_the_priors():
    import elfi_b200 as elfi
    dp = elfi.DeviceModelPrior(cases.six_model())
    res = elfi.Rejection(dp.model['d'], batch_size=50000, seed=3).sample(100000, quantile=1.0,
                                                                         bar=False)
    for name, case in zip(cases.SIX_NAMES, cases.SIX_PRIORS):
        v = res.samples[name]
        assert v.size == 100000
        assert ss.kstest(v, cases.frozen(*case).cdf).pvalue > 1e-3, name


def test_smc_with_device_model_prior():
    """SMC with device priors and proposals vs SMC with host priors and host proposals on the same
    six-parameter model; runs with one seed are identical, also in groups of two batches
    (distributed=False, max_parallel_batches=2: the single-rank side of the W-rank identity of
    DESIGN.md section 5), whose round 0 -- an even number of batches -- is the sequential one."""
    import elfi_b200 as elfi
    m = cases.six_model()
    dp = elfi.DeviceModelPrior(m)

    def run(**kw):
        return elfi.SMC(dp.model['d'], batch_size=20000, seed=5, device_proposal=dp, **kw).sample(
            4000, quantiles=[0.1, 0.3, 0.3], bar=False)
    res = run()
    assert len(res.populations) == 3
    assert np.isfinite(pr.joint_logpdf(dp.specs, res.samples_array)).all()
    ref = elfi.SMC(m['d'], batch_size=20000, seed=5).sample(4000, quantiles=[0.1, 0.3, 0.3],
                                                            bar=False)
    _posterior_check(res, ref, 'SMC')
    again = run()
    assert np.array_equal(res.samples_array, again.samples_array)
    assert np.array_equal(res.weights, again.weights)
    par = run(distributed=False, max_parallel_batches=2)
    par2 = run(distributed=False, max_parallel_batches=2)
    assert np.array_equal(par.samples_array, par2.samples_array)
    assert np.array_equal(par.weights, par2.weights)
    assert [p.threshold for p in par.populations] == [p.threshold for p in par2.populations]
    p0, q0 = res.populations[0], par.populations[0]
    assert p0.threshold == q0.threshold and p0.n_sim == q0.n_sim == 40000
    for name in cases.SIX_NAMES:
        assert np.array_equal(p0.outputs[name], q0.outputs[name])
    _posterior_check(par, ref, 'SMC in groups of two batches')


def test_adaptive_threshold_smc_with_device_model_prior():
    import elfi_b200 as elfi
    m = cases.six_model()
    dp = elfi.DeviceModelPrior(m)
    res = elfi.AdaptiveThresholdSMC(dp.model['d'], batch_size=20000, seed=4,
                                    device_proposal=dp).sample(2000, max_iter=4, bar=False)
    assert 2 <= len(res.populations) <= 4
    assert np.isfinite(pr.joint_logpdf(dp.specs, res.samples_array)).all()
    obs = dp.model.observed['sim'][0]
    assert np.all(np.abs(res.sample_means_array - obs) < 0.5), (res.sample_means_array, obs)


def test_gnk_stock_priors_cover_the_bespoke_proposal():
    """AdaptiveDistanceSMC on the throughput g-and-k model: priors written as stock
    Prior('uniform', 0, 10) with DeviceModelPrior vs the bespoke gnk.get_device_model() and
    gnk.DeviceProposal; the posterior means agree statistically."""
    import elfi_b200 as elfi
    from elfi_b200 import model as em
    from elfi_b200.examples import gnk
    n_obs = 64
    m = em.new_model()
    priors = [em.Prior('uniform', 0, 10, model=m, name=n) for n in ('A', 'B', 'g', 'k')]
    y_obs = gnk.GNK(3, 1, 2, .5, n_obs=n_obs, random_state=np.random.RandomState(7))
    em.Simulator(partial(gnk.gnk_device, n_obs=n_obs), *priors, observed=y_obs, name='GNK')
    em.AdaptiveDistance(em.Summary(gnk.ss_sorted, m['GNK'], name='ss_sorted'), name='d')
    dp = elfi.DeviceModelPrior(m)
    kw = dict(rounds=3, quantile=0.5, bar=False)
    res = elfi.AdaptiveDistanceSMC(dp.model['d'], batch_size=8000, seed=13,
                                   device_proposal=dp).sample(2000, **kw)
    mb, proposal = gnk.get_device_model(n_obs=n_obs, seed=7)
    ref = elfi.AdaptiveDistanceSMC(mb['d'], batch_size=8000, seed=13,
                                   device_proposal=proposal).sample(2000, **kw)
    assert len(res.populations) == len(ref.populations) == 3
    for pop in res.populations:
        for name in ('A', 'B', 'g', 'k'):
            assert pop.outputs[name].min() >= 0.0 and pop.outputs[name].max() <= 10.0
    _posterior_check(res, ref, 'g-and-k')
