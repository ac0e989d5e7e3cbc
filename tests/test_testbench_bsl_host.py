"""Lock-step BSL in the Testbench on the CPU double: the doubles of the two new entry points against
the existing doubles applied per group or per chain, lock-step against serial bit for bit, the
reference's Testbench golden in both run modes, the fallback rules and the argument checks."""
import numpy as np
import pytest
import torch

import abi_double
import bsl_chains_double
import bsl_double
import priors_double
import testbench_bsl_double
import elfi_b200 as elfi
from elfi_b200 import bsl, ops
from elfi_b200 import device as dev
from elfi_b200.examples import ma2

OBS_ENTRY = 'elfi_b200_synlik_obs_f64'
SIGMA = np.array([[.02, .01], [.01, .02]])
CASE = dict(repetitions=3, seed=156)
MK = dict(n_sim_round=200, feature_names=['MA2'])
SK = dict(n_samples=50, sigma_proposals=SIGMA, params0=np.array([.6, .2]))


@pytest.fixture
def double(cpu_double, monkeypatch):
    abi_double.install(monkeypatch, bsl_double.TABLE, bsl_chains_double.TABLE,
                                    priors_double.TABLE, testbench_bsl_double.TABLE)
    return cpu_double


def _model():
    return ma2.get_model(n_obs=50, true_params=[.6, .2], seed_obs=4)


def _testbench(method_kwargs, sample_kwargs, model=None, reps=CASE['repetitions'],
               seed=CASE['seed']):
    tb = elfi.Testbench(model=model or _model(), repetitions=reps, seed=seed, progress_bar=False)
    m = elfi.TestbenchMethod(method=bsl.BSL, name='BSL')
    m.set_method_kwargs(**method_kwargs)
    m.set_sample_kwargs(**sample_kwargs)
    tb.add_method(m)
    return tb, m


def _run(method_kwargs, sample_kwargs, lockstep, model=None, reps=CASE['repetitions'],
         double=None):
    tb, _ = _testbench(method_kwargs, sample_kwargs, model, reps)
    before = double.CALLS.count(OBS_ENTRY) if double is not None else 0
    tb.run(lockstep=lockstep)
    calls = double.CALLS.count(OBS_ENTRY) - before if double is not None else 0
    return tb.testbench_results[0]['results'], calls


@pytest.fixture
def logposteriors(monkeypatch):
    """state['logposterior'] of every BSL sampler when it extracts its result, in order."""
    kept = []
    extract = bsl.BSL.extract_result

    def keep(self):
        kept.append(np.array(self.state['logposterior']))
        return extract(self)
    monkeypatch.setattr(bsl.BSL, 'extract_result', keep)
    return kept


def assert_same_bsl(a, b):
    assert len(a) == len(b)
    for s, t in zip(a, b):
        assert list(s.samples_all) == list(t.samples_all)
        for k in s.samples_all:
            np.testing.assert_array_equal(s.samples_all[k], t.samples_all[k])
        for key in ('acc_rate', 'n_sim', 'burn_in'):
            assert getattr(s, key) == getattr(t, key), key
        for key in ('chains', 'acc_rates'):
            if key in s.meta or key in t.meta:
                np.testing.assert_array_equal(s.meta[key], t.meta[key])


# -- the entry-point doubles against the existing doubles -----------------------------------------
@pytest.mark.parametrize('kw', [dict(), dict(penalties=[0.0, 0.4]), dict(whitening=True),
                                dict(estimator='unbiased')])
def test_synlik_obs_double_is_the_double_per_group(double, kw):
    rs = np.random.RandomState(3)
    G, n, d = 5, 40, 4
    S = rs.randn(G, n, d) @ (np.eye(d) + 0.3 * rs.randn(d, d))
    S[2, 7, 1] = np.nan                          # a failure stays in its group
    wide = rs.randn(G, d + 3)
    Y = wide[:, :d]                              # gapped rows
    kw = dict(kw)
    if kw.pop('whitening', False):
        kw['whitening'] = np.eye(d) + 0.1 * rs.randn(d, d)
    W = kw.get('whitening')
    got = ops.synlik(S, dev.to_device(wide)[:, :d], **kw).cpu().numpy()
    assert double.CALLS[-1] == OBS_ENTRY
    for g in range(G):
        want = bsl_double.synlik(S[g], Y[g], kw.get('estimator', 'standard'), kw.get('penalties'),
                                 W)
        np.testing.assert_array_equal(got[g], want[0])
    assert np.all(np.isneginf(got[2]))


def test_synlik_obs_double_shared_row_and_routing(double, monkeypatch):
    rs = np.random.RandomState(4)
    G, n, d = 4, 30, 3
    S = rs.randn(G, n, d)
    y = rs.randn(d)
    strides = []

    def record(*args):
        strides.append(args[8])
        return testbench_bsl_double.synlik_obs_f64(*args)
    monkeypatch.setitem(testbench_bsl_double.TABLE, OBS_ENTRY, record)
    shared = ops.synlik(S, dev.to_device(y)[None].expand(G, d)).cpu().numpy()
    assert strides == [0]                        # an expanded row is passed as ld_y = 0
    np.testing.assert_array_equal(shared, bsl_double.synlik(S, y))
    # d values, (d,) or (1, d), keep the entry point of one shared row (which the BSL doubles
    # intercept), whatever G is
    for yy in (y, y[None], dev.to_device(y)[None]):
        np.testing.assert_array_equal(ops.synlik(S, yy).cpu().numpy(), shared)
        assert double.CALLS[-1] == 'elfi_b200_synlik_f64'
    assert strides == [0]
    with pytest.raises(Exception, match='observation stride'):
        testbench_bsl_double.synlik_obs_f64(None, 0, d, n * d, G, n, d, 0, 2, None, 0, None, 0,
                                            0, None)


def _step_case(p, bounds):
    rs = np.random.RandomState(7 + p)
    lo = rs.uniform(-1.5, -0.5, p)
    specs = np.array([[0, lo[a], rs.uniform(1.5, 3.0), 0, 0] for a in range(p)])
    x0 = specs[:, 1] + 0.5 * specs[:, 2]
    bnd = None
    if bounds:
        bnd = np.column_stack([specs[:, 1] - 1.0, specs[:, 1] + specs[:, 2] + 1.0])
        bnd[0, 0] = -np.inf
    return rs, specs, x0, ops.bsl_mh_tables(specs, np.eye(p) * 0.5, None, bnd)


def _state(x, C, n, p):
    return dict(prop=dev.to_device(x), chains=dev.zeros((C, n, p)), logpost=dev.zeros((C, n)),
                n_acc=dev.zeros((C,), dtype=torch.int64))


@pytest.mark.parametrize('bounds', [False, True])
@pytest.mark.parametrize('lanes', [None, [3, 0, 6, 1]])
def test_keyed_step_double_is_the_step_per_chain(double, bounds, lanes):
    p, C, n, b = 2, 4, 6, 3
    rs, specs, x0, tables = _step_case(p, bounds)
    keys = np.array([11, 2 ** 40 + 5, 11, 987654321], dtype=np.int64)
    starts = np.tile(x0, (C, 1)) + 0.05 * rs.randn(C, p)
    lls = rs.randn(n, C) * 3.0 - 50.0
    at = np.arange(C) if lanes is None else np.array(lanes)
    keyed = _state(starts, C, n, p)
    keyed['prop_lp'] = ops.prior_logpdf(keyed['prop'], specs)
    rows = dev.zeros((p, C * b))
    lane_arg = None if lanes is None else dev.to_device(np.array(lanes), dtype=torch.int64)
    for t in range(n):
        ops.bsl_mh_step(tables, t, dev.to_device(lls[t]), keyed['prop'], keyed['prop_lp'],
                        keyed['chains'], keyed['logpost'], keyed['n_acc'], rows,
                        dev.to_device(keys, dtype=torch.int64), 1, lanes=lane_arg)
    assert double.CALLS[-1] == 'elfi_b200_bsl_mh_step_keyed_f64'
    for c in range(C):
        # slot c is the chain at slot at[c] of an unkeyed step seeded with keys[c]
        L = int(at[c]) + 1
        one = _state(np.tile(starts[c], (L, 1)), L, n, p)
        one['prop_lp'] = ops.prior_logpdf(one['prop'], specs)
        rows1 = dev.zeros((p, L * b))
        for t in range(n):
            ops.bsl_mh_step(tables, t, dev.to_device(np.full(L, lls[t, c])), one['prop'],
                            one['prop_lp'], one['chains'], one['logpost'], one['n_acc'], rows1,
                            int(keys[c]), 1)
        for k in ('chains', 'logpost', 'n_acc', 'prop', 'prop_lp'):
            np.testing.assert_array_equal(keyed[k].cpu().numpy()[c], one[k].cpu().numpy()[L - 1])
        np.testing.assert_array_equal(rows.cpu().numpy()[:, c * b:(c + 1) * b],
                                      rows1.cpu().numpy()[:, (L - 1) * b:L * b])
    # the keys make a difference: slots 0 and 2 share a key, not a lane unless lanes say so
    ch = keyed['chains'].cpu().numpy()
    assert not np.array_equal(ch[0], ch[1])


def test_argument_errors(double):
    S = np.random.RandomState(0).randn(3, 20, 4)
    with pytest.raises(ValueError, match='y has shape'):
        ops.synlik(S, np.zeros((2, 4)))
    with pytest.raises(ValueError, match='y has 3 values'):
        ops.synlik(S, np.zeros(3))
    p, C, n, b = 2, 3, 4, 2
    _, specs, x0, tables = _step_case(p, False)
    st = _state(np.tile(x0, (C, 1)), C, n, p)
    st['prop_lp'] = ops.prior_logpdf(st['prop'], specs)
    args = (tables, 0, dev.zeros((C,)), st['prop'], st['prop_lp'], st['chains'], st['logpost'],
            st['n_acc'], dev.zeros((p, C * b)))
    with pytest.raises(ValueError, match='keys'):
        ops.bsl_mh_step(*args, dev.to_device(np.arange(C + 1), dtype=torch.int64))
    with pytest.raises(ValueError, match='keys'):
        ops.bsl_mh_step(*args, dev.to_device(np.arange(C), dtype=torch.float64))
    with pytest.raises(ValueError, match='lanes'):
        ops.bsl_mh_step(*args, dev.to_device(np.arange(C), dtype=torch.int64),
                        lanes=dev.to_device(np.arange(C + 1), dtype=torch.int64))
    with pytest.raises(ValueError, match='lanes'):
        ops.bsl_mh_step(*args, 5, lanes=dev.to_device(np.arange(C), dtype=torch.int64))


# -- lock-step against serial, bit for bit --------------------------------------------------------
LIKELIHOODS = {
    'default': ({}, {}),
    'unbiased': (dict(likelihood=bsl.unbiased_likelihood()), {}),
    'whitened_warton': ('whitened', {}),
    'bounded': ({}, dict(burn_in=10, logit_transform_bound=[[-2., 2.], [-1., 1.]])),
    'two_chains': ({}, dict(n_chains=2, params0=np.array([[.6, .2], [.3, .1]]))),
}


@pytest.mark.parametrize('case', list(LIKELIHOODS))
def test_lockstep_equals_serial(double, logposteriors, case):
    mk, sk = LIKELIHOODS[case]
    if mk == 'whitened':
        W = np.diag(1.0 / np.linspace(0.5, 1.5, 50))
        mk = dict(likelihood=bsl.standard_likelihood(shrinkage='warton', penalty=0.3,
                                                     whitening=W))
    mk, sk = dict(MK, **mk), dict(SK, **sk)
    lock, n_lock = _run(mk, sk, True, double=double)
    lock_lp = logposteriors[:]
    del logposteriors[:]
    serial, n_serial = _run(mk, sk, False, double=double)
    assert_same_bsl(lock, serial)
    assert len(lock_lp) == len(logposteriors) == CASE['repetitions']
    for a, b in zip(lock_lp, logposteriors):
        np.testing.assert_array_equal(a, b)
    assert n_serial == 0
    # one call per lock-step iteration: as many as the repetition that simulates the most rounds
    C = sk.get('n_chains', 1)
    rounds = [s.n_sim // (MK['n_sim_round'] * C) for s in serial]
    assert n_lock == max(rounds)
    if case == 'default':
        assert len(set(rounds)) > 1              # ragged progress


def test_throughput_lockstep_equals_serial(double, logposteriors, monkeypatch):
    m, dp = ma2.get_uniform_device_model(n_obs=20, seed_obs=4)
    mk = dict(n_sim_round=60, feature_names=['MA2'], batch_size=30, device_proposal=dp)
    sk = dict(n_samples=12, sigma_proposals=np.diag([.05, .05]), params0=[.6, .2], burn_in=2,
              n_chains=2, logit_transform_bound=[[-2., 2.], [-1., 1.]])
    reads = []
    to_host = dev.to_host
    monkeypatch.setattr(dev, 'to_host', lambda x: reads.append(tuple(np.shape(x))) or to_host(x))
    del double.CALLS[:]
    lock, _ = _run(mk, sk, True, model=m)
    calls = list(double.CALLS)
    lock_reads = reads[:]
    lock_lp = logposteriors[:]
    del logposteriors[:]
    serial, _ = _run(mk, sk, False, model=m)
    assert_same_bsl(lock, serial)
    for a, b in zip(lock_lp, logposteriors):
        np.testing.assert_array_equal(a, b)
    assert calls.count('elfi_b200_bsl_mh_step_keyed_f64') == 12
    assert calls.count(OBS_ENTRY) == 12
    assert 'elfi_b200_bsl_mh_step_f64' not in calls
    # one read of the first round's R C log-likelihoods; the rest is extract_result's (3 arrays
    # per repetition) and the Testbench's own set-up
    assert lock_reads.count((3 * 2,)) == 1
    assert all(r.n_sim == 12 * 2 * 60 for r in lock)


# -- the reference's Testbench --------------------------------------------------------------------
@pytest.mark.parametrize('lockstep', [True, False])
def test_matches_reference_golden(double, logposteriors, golden, lockstep):
    g = golden('testbench_bsl')
    tb, _ = _testbench(MK, SK)
    np.testing.assert_array_equal(tb.observations, g['observations'])
    np.testing.assert_array_equal(tb.method_seed_list[0], g['seeds'])
    for t in ('t1', 't2'):
        np.testing.assert_array_equal(tb.reference_parameter[t], g['ref_' + t])
    tb.run(lockstep=lockstep)
    for r, s in enumerate(tb.testbench_results[0]['results']):
        key = 'r{}_'.format(r)
        np.testing.assert_array_equal(np.column_stack([s.samples_all['t1'], s.samples_all['t2']]),
                                      g[key + 'samples_all'])
        assert s.n_sim == int(g[key + 'nsim'])
        assert s.acc_rate == float(g[key + 'acc_rate'])
        lp = g[key + 'logposterior']
        assert np.all(np.abs(logposteriors[r] - lp) <= 1e-9 * (1 + np.abs(lp)))
    assert len({int(g['r{}_nsim'.format(r)]) for r in range(3)}) == 3


# -- what runs serially ---------------------------------------------------------------------------
@pytest.mark.parametrize('case', ['host_likelihood', 'pool', 'fit_kwargs', 'other_method'])
def test_fallback_runs_serially(double, case):
    mk = dict(MK)
    tb, method = _testbench(mk, dict(SK, n_samples=5), reps=2)
    if case == 'host_likelihood':
        method.attributes['method_kwargs'] = dict(mk, likelihood=bsl_double.synlik)
    elif case == 'pool':
        method.attributes['method_kwargs'] = dict(mk, pool=elfi.OutputPool(['MA2']))
    elif case == 'fit_kwargs':
        method.attributes['fit_kwargs'] = dict(n_evidence=10)
    else:
        method.attributes['callable'] = elfi.Rejection
    assert not tb._lockstep_bsl_applies(method)
    if case == 'host_likelihood':
        before = double.CALLS.count(OBS_ENTRY)
        tb.run()
        assert double.CALLS.count(OBS_ENTRY) == before
        assert len(tb.testbench_results[0]['results']) == 2
    _, plain = _testbench(MK, SK)
    assert tb._lockstep_bsl_applies(plain)
    plain.attributes['method_kwargs'] = dict(MK, likelihood=bsl.unbiased_likelihood())
    assert tb._lockstep_bsl_applies(plain)
