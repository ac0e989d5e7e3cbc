"""Lock-step BSL in the Testbench on the device: elfi_b200_synlik_obs_f64 against G separate
ops.synlik calls and elfi_b200_bsl_mh_step_keyed_f64 against separate single-sampler steps, bit for
bit; lock-step against serial on the host MA2 model and the device MA2 model in parity and
throughput mode; the reference's Testbench golden in both run modes; and the device-to-host reads
of a lock-step run."""
import ctypes

import numpy as np
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

from elfi_b200 import _lib, ops
from elfi_b200 import device as dev
from elfi_b200.examples import ma2

from test_testbench_bsl_host import (MK, SK, _run, _testbench, assert_same_bsl,  # noqa: F401
                                     logposteriors)  # a fixture

pytestmark = pytest.mark.gpu

# (d, n, G, extra, Y layout): G = 1 and 7 split their rows over several CTAs where n > 256, G = 64
# at d >= 145 walks its chunks inside one CTA, and n <= 256 has a single chunk
SYNLIK_CASES = [
    (1, 300, 7, 'plain', 'gapped'), (1, 5000, 64, 'penalties', 'shared'),
    (33, 2000, 7, 'penalties', 'gapped'), (33, 257, 64, 'whitening', 'shared'),
    (145, 5000, 7, 'unbiased', 'gapped'), (145, 1000, 64, 'penalties', 'gapped'),
    (145, 256, 64, 'plain', 'gapped'),
    (160, 5000, 64, 'whitening', 'gapped'), (160, 200, 1, 'plain', 'gapped'),
    (160, 5000, 1, 'penalties', 'shared'), (160, 3000, 7, 'whitening', 'shared'),
]


def _synlik_case(d, n, G, extra, layout):
    rs = np.random.RandomState(d * 7 + n + G)
    A = np.eye(d) + 0.2 * rs.randn(d, d) / np.sqrt(d)
    S = torch.tensor(rs.randn(G, n, d) @ A + rs.randn(d), device='cuda')
    if G >= 7:
        S[1, 3, 0] = float('nan')                  # a non-finite input: -inf in group 1 only
        if d >= 2:
            S[2, :, 1] = S[2, :, 0]                # a duplicated column: -inf in group 2 only
                                                   # (at penalty 0)
    kw = {}
    if extra == 'penalties':
        kw['penalties'] = [0.0, 0.25, 1.0]
    elif extra == 'whitening':
        kw['whitening'] = torch.tensor(np.eye(d) + 0.05 * rs.randn(d, d) / np.sqrt(d),
                                       device='cuda')
    elif extra == 'unbiased':
        kw['estimator'] = 'unbiased'
    centre = S.nan_to_num().mean(dim=1)
    if layout == 'gapped':
        wide = torch.tensor(rs.randn(G, d + 5), device='cuda')
        wide[:, :d] = centre + 0.1
        Y = wide[:, :d]
    else:
        Y = (centre[0] + 0.1)[None].expand(G, d)
    return S, Y, kw


def _synlik_obs(S, Y, penalties=None, whitening=None, estimator='standard'):
    """elfi_b200_synlik_obs_f64 called directly, ld_y = Y.stride(0) (ops.synlik takes a single
    row, G = 1 included, to elfi_b200_synlik_f64)."""
    G, n, d = S.shape
    pen = None if penalties is None else np.asarray(penalties, dtype=np.float64)
    K = 0 if pen is None else pen.size
    out = torch.empty((G, K) if K else (G,), dtype=torch.float64, device='cuda')
    _lib.call('elfi_b200_synlik_obs_f64', dev.context(), dev.ptr(S), S.stride(1), S.stride(0), G,
              n, d, dev.ptr(Y), Y.stride(0), dev.ptr(whitening), ops.SYNLIK_ESTIMATORS[estimator],
              None if pen is None else ctypes.c_void_p(pen.ctypes.data), K, dev.ptr(out),
              dev.stream_ptr())
    return out.cpu().numpy()


@pytest.mark.parametrize('d,n,G,extra,layout', SYNLIK_CASES)
def test_synlik_obs_is_separate_calls(d, n, G, extra, layout):
    S, Y, kw = _synlik_case(d, n, G, extra, layout)
    got = ops.synlik(S, Y, **kw).cpu().numpy()
    want = np.stack([ops.synlik(S[g], Y[g].contiguous(), **kw).cpu().numpy()[0]
                     for g in range(G)])
    np.testing.assert_array_equal(got, want)
    np.testing.assert_array_equal(_synlik_obs(S, Y, **kw), want)
    assert np.isfinite(got[0]).all()
    if G >= 7:
        assert np.isneginf(got[1]).all() and np.isfinite(got[3:]).all()
        if d >= 2:
            # singular without shrinkage; a Warton penalty above 0 makes it positive definite
            assert np.isneginf(np.reshape(got[2], -1)[0])
    if layout == 'shared':
        # one row for every group is what the one-observation entry point computes
        np.testing.assert_array_equal(got, ops.synlik(S, Y[0].contiguous(), **kw).cpu().numpy())
    again = ops.synlik(S, Y, **kw).cpu().numpy()
    np.testing.assert_array_equal(again, got)


def _kernels(fn):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def test_split_and_walk_forms_both_run():
    """Without whitening, synlik_reduce_kernel runs only in the split form."""
    S, Y, _ = _synlik_case(160, 5000, 64, 'plain', 'gapped')
    walk = _kernels(lambda: ops.synlik(S, Y))
    split = _kernels(lambda: ops.synlik(S[5], Y[5].contiguous()))
    if any('synlik_factor_kernel' in k for k in walk + split):   # the trace kept the kernels
        assert not any('synlik_reduce_kernel' in k for k in walk)
        assert any('synlik_reduce_kernel' in k for k in split)


def _specs(p, rs):
    lo = rs.uniform(-1.5, -0.5, p)
    return np.array([[0, lo[a], rs.uniform(1.5, 3.0), 0, 0] for a in range(p)])


def _state(x):
    C, p = x.shape
    prop = torch.tensor(x, device='cuda')
    return dict(prop=prop, chains=torch.zeros((C, 10, p), dtype=torch.float64, device='cuda'),
                logpost=torch.zeros((C, 10), dtype=torch.float64, device='cuda'),
                n_acc=torch.zeros(C, dtype=torch.int64, device='cuda'))


@pytest.mark.parametrize('p', [2, 5])
@pytest.mark.parametrize('bounds', [False, True])
@pytest.mark.parametrize('lanes', [None, 'scattered'])
def test_keyed_step_is_separate_steps(p, bounds, lanes):
    rs = np.random.RandomState(p + 10 * bounds)
    specs = _specs(p, rs)
    bnd = None
    if bounds:
        bnd = np.column_stack([specs[:, 1] - 1.0, specs[:, 1] + specs[:, 2] + 1.0])
        bnd[::2, 1] = np.inf
    tables = ops.bsl_mh_tables(specs, np.eye(p) * 0.8, None, bnd)
    C, n, b = 12, 10, 4
    keys = rs.randint(0, 2 ** 32 - 1, size=C).astype(np.int64)
    keys[3] = keys[0]
    at = np.arange(C) if lanes is None else rs.permutation(40)[:C]
    starts = specs[:, 1] + 0.5 * specs[:, 2] + 0.05 * rs.randn(C, p)
    lls = rs.randn(n, C) * 3.0 - 50.0
    keyed = _state(starts)
    keyed['prop_lp'] = ops.prior_logpdf(keyed['prop'], specs)
    rows = torch.zeros((p, C * b), dtype=torch.float64, device='cuda')
    key_t = torch.tensor(keys, device='cuda')
    lane_t = None if lanes is None else torch.tensor(at, device='cuda')
    for t in range(n):
        ops.bsl_mh_step(tables, t, torch.tensor(lls[t], device='cuda'), keyed['prop'],
                        keyed['prop_lp'], keyed['chains'], keyed['logpost'], keyed['n_acc'], rows,
                        key_t, 2, lanes=lane_t)
    for c in range(C):
        # chain c alone at slot at[c] of an unkeyed step under seed keys[c]
        L = int(at[c]) + 1
        one = _state(np.tile(starts[c], (L, 1)))
        one['prop_lp'] = ops.prior_logpdf(one['prop'], specs)
        rows1 = torch.zeros((p, L * b), dtype=torch.float64, device='cuda')
        for t in range(n):
            ops.bsl_mh_step(tables, t, torch.full((L,), lls[t, c], dtype=torch.float64,
                                                  device='cuda'),
                            one['prop'], one['prop_lp'], one['chains'], one['logpost'],
                            one['n_acc'], rows1, int(keys[c]), 2)
        for k in ('chains', 'logpost', 'n_acc', 'prop', 'prop_lp'):
            np.testing.assert_array_equal(keyed[k][c].cpu().numpy(), one[k][L - 1].cpu().numpy())
        np.testing.assert_array_equal(rows[:, c * b:(c + 1) * b].cpu().numpy(),
                                      rows1[:, (L - 1) * b:L * b].cpu().numpy())
    moved = (keyed['chains'][:, 1:] != keyed['chains'][:, :-1]).any(dim=2)
    assert moved.any() and not moved.all()


# -- lock-step against serial ---------------------------------------------------------------------
def _models():
    um, dp = ma2.get_uniform_device_model(n_obs=50, true_params=[.6, .2], seed_obs=4)
    return {
        'host': (ma2.get_model(n_obs=50, true_params=[.6, .2], seed_obs=4), {}),
        'device': (ma2.get_device_model(n_obs=50, true_params=[.6, .2], seed_obs=4), {}),
        'throughput': (um, dict(device_proposal=dp)),
    }


@pytest.mark.parametrize('model', ['host', 'device', 'throughput'])
@pytest.mark.parametrize('reps,chains', [(1, 1), (4, 1), (4, 2)])
def test_lockstep_equals_serial(logposteriors, model, reps, chains):
    m, mk = _models()[model]
    mk = dict(MK, **mk)
    sk = dict(SK, n_samples=30)
    if chains > 1:
        sk.update(n_chains=chains, params0=np.array([[.6, .2], [.3, .1]]),
                  logit_transform_bound=[[-2., 2.], [-1., 1.]], burn_in=5)
    lock, _ = _run(mk, sk, True, model=m, reps=reps)
    lock_lp = logposteriors[:]
    del logposteriors[:]
    serial, _ = _run(mk, sk, False, model=m, reps=reps)
    assert_same_bsl(lock, serial)
    assert len(lock_lp) == len(logposteriors) == reps
    for a, b in zip(lock_lp, logposteriors):
        np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize('lockstep', [True, False])
def test_matches_reference_golden(logposteriors, golden, lockstep):
    g = golden('testbench_bsl')
    tb, _ = _testbench(MK, SK)
    np.testing.assert_array_equal(tb.observations, g['observations'])
    np.testing.assert_array_equal(tb.method_seed_list[0], g['seeds'])
    tb.run(lockstep=lockstep)
    for r, s in enumerate(tb.testbench_results[0]['results']):
        key = 'r{}_'.format(r)
        np.testing.assert_array_equal(np.column_stack([s.samples_all['t1'], s.samples_all['t2']]),
                                      g[key + 'samples_all'])
        assert s.n_sim == int(g[key + 'nsim'])
        assert s.acc_rate == float(g[key + 'acc_rate'])
        lp = g[key + 'logposterior']
        assert np.all(np.abs(logposteriors[r] - lp) <= 1e-9 * (1 + np.abs(lp)))


# -- device-to-host reads -------------------------------------------------------------------------
def _d2h_copies(fn):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events()
               if e.device_type == torch.autograd.DeviceType.CUDA and 'DtoH' in e.name)


@pytest.mark.parametrize('reps', [2, 6])
def test_reads_per_iteration(reps):
    """Parity mode: one read per lock-step iteration whatever R is (the difference of 20 and 10
    iterations, so the reads around the run cancel).  Throughput mode: the same count at 10 and
    20 iterations, so no iteration reads."""
    counts = {}
    m_dev = ma2.get_device_model(n_obs=50, true_params=[.6, .2], seed_obs=4)
    um, dp = ma2.get_uniform_device_model(n_obs=50, true_params=[.6, .2], seed_obs=4)
    for mode, m, mk in (('parity', m_dev, {}), ('throughput', um, dict(device_proposal=dp))):
        for n in (10, 20):
            # a narrow proposal that stays inside the triangular prior: every iteration simulates
            tb, _ = _testbench(dict(MK, **mk), dict(SK, n_samples=n,
                                                    sigma_proposals=np.diag([1e-6, 1e-6])),
                               model=m, reps=reps)
            counts[mode, n] = _d2h_copies(lambda: tb.run(lockstep=True))
    if counts['parity', 20] or counts['throughput', 20]:         # the trace kept the copies
        assert counts['parity', 20] - counts['parity', 10] == 10
        assert counts['throughput', 20] == counts['throughput', 10]
