"""Testbench on the CPU: the reference's tests/unit/test_testbench.py restated, seeds, observations
and reference parameters against the reference's golden, the NumPy double of the segmented entry
points against a direct statement, lock-step against serial, and the rules that send a method
down the serial path."""
import numpy as np
import pytest
import scipy.spatial.distance as ssd

import elfi_b200 as elfi
from elfi_b200 import device as dev
from elfi_b200 import ops
from elfi_b200.examples import ma2 as exma2

import abi_double
import testbench_double

SEG = ('elfi_b200_dist_seg_f64', 'elfi_b200_topn_merge_seg_f64')
CASE = dict(seed_obs=4, repetitions=3, seed=156)
REF_PARAM = {'t1': np.array([0.6]), 't2': np.array([0.2])}
METHODS = [
    ('Rejection', dict(discrepancy_name='d', batch_size=500), dict(n_samples=500)),
    ('Rejection', dict(discrepancy_name='d', batch_size=500), dict(n_samples=100, n_sim=2000)),
    ('Rejection', dict(discrepancy_name='d', batch_size=500), dict(n_samples=50, threshold=0.5)),
    ('SMC', dict(discrepancy_name='d', batch_size=500), dict(n_samples=100,
                                                            thresholds=[2.0, 1.0])),
]


@pytest.fixture
def tb_double(cpu_double, monkeypatch):
    abi_double.install(monkeypatch, testbench_double.TABLE)
    return cpu_double


@pytest.fixture
def ma2():
    return exma2.get_model()


def golden_testbench(golden, case, methods=range(4)):
    g = golden('testbench')
    m = exma2.get_model(seed_obs=CASE['seed_obs'])
    given = {}
    if case == 'obs':
        given['observations'] = g['obs_observations'][:1].copy()
    elif case == 'param':
        given['reference_parameter'] = {k: v.copy() for k, v in REF_PARAM.items()}
    tb = elfi.Testbench(model=m, repetitions=CASE['repetitions'], seed=CASE['seed'],
                        progress_bar=False, **given)
    for k, (cls, mk, sk) in enumerate(METHODS):
        if k not in methods:
            tb._get_seeds(n_rep=tb.repetitions)     # keep the seed stream of the reference
            continue
        method = elfi.TestbenchMethod(method=getattr(elfi, cls), name='m{}'.format(k))
        method.set_method_kwargs(**mk)
        method.set_sample_kwargs(bar=False, **sk)
        tb.add_method(method)
    return g, tb


# -- the reference's tests/unit/test_testbench.py ------------------------------------------------
def test_testbenchmethod_init():
    method = elfi.TestbenchMethod(method=elfi.SMC, name="SMC_1")
    method.set_method_kwargs(discrepancy_name='d', batch_size=50)
    method.set_sample_kwargs(n_samples=100, thresholds=[2.0, 1.0], bar=False)
    attr = method.get_method()
    assert attr['name'] == "SMC_1"
    assert attr['method_kwargs']['batch_size'] == 50
    assert attr['sample_kwargs']['n_samples'] == 100
    assert elfi.TestbenchMethod(method=elfi.Rejection).attributes['name'] == 'Rejection'


def test_testbench_init_param_reps(ma2):
    testbench = elfi.Testbench(model=ma2, repetitions=5, seed=99, progress_bar=False)
    for _, values in testbench.reference_parameter.items():
        assert values.size == 5


def test_testbench_init_given_params(ma2):
    ref_params = ma2.generate(batch_size=1, outputs=['t1', 't2'])
    testbench = elfi.Testbench(model=ma2, reference_parameter=ref_params, repetitions=5, seed=99,
                               progress_bar=False)
    for _, values in testbench.reference_parameter.items():
        assert np.all(values == values[0])
        assert values.size == 5


def test_testbench_init_obs_reps(ma2):
    testbench = elfi.Testbench(model=ma2, repetitions=5, seed=99, progress_bar=False)
    assert len(testbench.observations) == 5


def test_testbench_init_given_obs(ma2):
    obs = ma2.generate(batch_size=1, outputs=['MA2'])
    testbench = elfi.Testbench(model=ma2, observations=obs, repetitions=5, seed=99,
                               progress_bar=False)
    assert len(testbench.observations) == 5
    assert np.all([a == b for a, b in zip([obs], testbench.observations)])


def test_testbench_execution(tb_double, ma2):
    method1 = elfi.TestbenchMethod(method=elfi.Rejection, name='Rejection_1')
    method1.set_method_kwargs(discrepancy_name='d', batch_size=500)
    method1.set_sample_kwargs(n_samples=500, bar=False)
    method2 = elfi.TestbenchMethod(method=elfi.Rejection, name='Rejection_2')
    method2.set_method_kwargs(discrepancy_name='d', batch_size=500)
    method2.set_sample_kwargs(n_samples=500, quantile=0.5, bar=False)
    testbench = elfi.Testbench(model=ma2, repetitions=3, seed=156, progress_bar=False)
    testbench.add_method(method1)
    testbench.add_method(method2)
    testbench.run()
    sample_mean_differences = testbench.parameterwise_sample_mean_differences()
    assert len(sample_mean_differences) == 2
    assert len(sample_mean_differences['Rejection_1']) == 2
    assert len(sample_mean_differences['Rejection_1']['t1']) == 3
    results = testbench.get_testbench_results()
    assert set(results) == {'testcases', 'results'}
    assert set(results['testcases']) == {'model', 'observations', 'reference_parameter',
                                         'reference_posterior'}
    assert [r['method'] for r in results['results']] == ['Rejection_1', 'Rejection_2']
    assert all(len(r['results']) == 3 for r in results['results'])


def test_testbench_seeding(ma2):
    testbench1 = elfi.Testbench(model=ma2, repetitions=2, seed=100, progress_bar=False)
    testbench2 = elfi.Testbench(model=ma2, repetitions=2, seed=100, progress_bar=False)
    assert len(testbench1.observations) == len(testbench2.observations)
    assert np.all([a == b for a, b in zip(testbench1.observations, testbench2.observations)])


def test_progress_bar_is_accepted(tb_double, ma2, capsys):
    tb = elfi.Testbench(model=ma2, repetitions=2, seed=1, progress_bar=True)
    method = elfi.TestbenchMethod(method=elfi.Rejection)
    method.set_method_kwargs(discrepancy_name='d', batch_size=100)
    method.set_sample_kwargs(n_samples=10, bar=False)
    tb.add_method(method)
    tb.run()
    assert 'Progress' in capsys.readouterr().out
    assert tb._compare_sample_results() is None and tb._retrodiction() is None


# -- the reference's seeds and simulated data ----------------------------------------------------
@pytest.mark.parametrize('case', ['sim', 'obs', 'param'])
def test_seeds_observations_and_parameters_match_golden(golden, case):
    g, tb = golden_testbench(golden, case)
    np.testing.assert_array_equal(tb.observations, g[case + '_observations'])
    assert tb.observations.dtype == g[case + '_observations'].dtype
    if case == 'obs':
        assert tb.reference_parameter is None
    else:
        for t in ('t1', 't2'):
            np.testing.assert_array_equal(tb.reference_parameter[t], g['{}_ref_{}'.format(case, t)])
    for k in range(len(METHODS)):
        np.testing.assert_array_equal(tb.method_seed_list[k], g['{}_m{}_seeds'.format(case, k)])
        assert tb.method_seed_list[k].dtype == np.uint32


@pytest.mark.parametrize('lockstep', [True, False])
def test_rejection_matches_golden_on_the_double(tb_double, golden, lockstep):
    g, tb = golden_testbench(golden, 'sim', methods=(0, 1, 2))
    tb.run(lockstep=lockstep)
    for k, res in enumerate(tb.testbench_results):
        for r, s in enumerate(res['results']):
            key = 'sim_m{}_r{}_'.format(k, r)
            for t in ('t1', 't2'):
                np.testing.assert_array_equal(s.samples[t], g[key + t])
            np.testing.assert_array_equal(s.discrepancies, g[key + 'd'])
            assert s.n_sim == int(g[key + 'nsim'])
    smd = tb.parameterwise_sample_mean_differences()
    for k in range(3):
        for t in ('t1', 't2'):
            np.testing.assert_array_equal(smd['m{}'.format(k)][t], g['sim_m{}_smd_{}'.format(k, t)])
    # m0: 100 batches (quantile 0.01 of 500 samples), m1: 4 batches, m2 (threshold): serial
    assert tb_double.CALLS.count('elfi_b200_dist_seg_f64') == (104 if lockstep else 0)


# -- the double against a direct statement -------------------------------------------------------
@pytest.mark.parametrize('metric,p', [('euclidean', 2.0), ('sqeuclidean', 2.0), ('cityblock', 2.0),
                                      ('chebyshev', 2.0), ('minkowski', 3.0)])
def test_dist_seg_double_matches_cdist(tb_double, metric, p):
    rng = np.random.RandomState(0)
    R, B, D = 5, 37, 6
    S = rng.randn(R * B, D + 3)[:, :D]          # strided rows
    obs = rng.randn(R, D + 2)[:, :D]
    S[3, 1] = np.nan
    S[40, 0] = np.inf
    d = ops.dist_seg(S, obs, metric, p).cpu().numpy()
    kw = {'p': p} if metric == 'minkowski' else {}
    want = np.concatenate([ssd.cdist(S[r * B:(r + 1) * B], obs[r:r + 1], metric, **kw)[:, 0]
                           for r in range(R)])
    np.testing.assert_array_equal(d, want)
    assert tb_double.CALLS[-1] == 'elfi_b200_dist_seg_f64'


def test_dist_seg_rejects_what_it_does_not_compute(tb_double):
    with pytest.raises(ValueError):
        ops.dist_seg(np.zeros((6, 2)), np.zeros((4, 2)))       # 6 rows are not 4 segments
    with pytest.raises(ValueError):
        ops.dist_seg(np.zeros((6, 2)), np.zeros((3, 2)), 'cosine')
    with pytest.raises(ValueError):
        ops.dist_seg(np.zeros((6, 3)), np.zeros((3, 2)))


@pytest.mark.parametrize('nA', [0, 3, 8])
def test_topn_merge_seg_double_matches_argsort(tb_double, nA):
    rng = np.random.RandomState(1)
    R, nB, n_keep = 4, 9, min(8, nA + 9)
    ka = np.round(rng.rand(R, nA) * 4) / 4          # ties
    kb = np.round(rng.rand(R, nB) * 4) / 4
    kb[0, 2], kb[1, 0], kb[2, 5] = np.nan, np.inf, -np.inf
    widths = [1, 3]
    A = [rng.randn(R, nA, w) for w in widths]
    Bs = [rng.randn(R, nB, w) for w in widths]
    tops = ops.merge_topn_seg(
        [dev.to_device(a[:, :, 0] if w == 1 else a) for a, w in zip(A, widths)],
        [dev.to_device(b[:, :, 0] if w == 1 else b) for b, w in zip(Bs, widths)],
        dev.to_device(ka), dev.to_device(kb), n_keep)
    for r in range(R):
        order = np.argsort(np.concatenate([ka[r], kb[r]]), kind='stable')[:n_keep]
        for top, a, b, w in zip(tops, A, Bs, widths):
            want = np.concatenate([a[r], b[r]])[order]
            got = top[r].cpu().numpy().reshape(n_keep, w)
            np.testing.assert_array_equal(got, want)


# -- lock-step against serial --------------------------------------------------------------------
def run_both(model, method_kwargs, sample_kwargs, reps=3, seed=7, method=None):
    out = []
    for lockstep in (True, False):
        tb = elfi.Testbench(model=model, repetitions=reps, seed=seed, progress_bar=False)
        m = elfi.TestbenchMethod(method=method or elfi.Rejection)
        m.set_method_kwargs(**method_kwargs)
        m.set_sample_kwargs(bar=False, **sample_kwargs)
        tb.add_method(m)
        tb.run(lockstep=lockstep)
        out.append(tb.testbench_results[0]['results'])
    return out


def assert_same_samples(a, b):
    assert len(a) == len(b)
    for s, t in zip(a, b):
        assert list(s.outputs) == list(t.outputs)
        for k in s.outputs:
            np.testing.assert_array_equal(np.asarray(s.outputs[k]), np.asarray(t.outputs[k]))
        for key in ('n_sim', 'n_batches', 'threshold', 'accept_rate', 'seed', 'method_name'):
            assert getattr(s, key) == getattr(t, key), key


@pytest.mark.parametrize('sample_kwargs', [dict(n_samples=40, quantile=0.1),
                                           dict(n_samples=30, n_sim=1000)])
def test_lockstep_equals_serial_with_extra_outputs(tb_double, sample_kwargs):
    m = exma2.get_model(seed_obs=4)
    calls = len(tb_double.CALLS)
    lock, serial = run_both(m, dict(discrepancy_name='d', batch_size=100,
                                    output_names=['S1', 'S2']), sample_kwargs)
    assert 'elfi_b200_topn_merge_seg_f64' in tb_double.CALLS[calls:]
    assert_same_samples(lock, serial)
    assert 'S1' in lock[0].outputs


def test_lockstep_other_metric_and_single_repetition(tb_double):
    m = exma2.get_model(seed_obs=4)
    elfi.Distance('cityblock', m['S1'], m['S2'], name='d1')
    lock, serial = run_both(m, dict(discrepancy_name='d1', batch_size=64),
                            dict(n_samples=20, quantile=0.05), reps=1)
    assert 'elfi_b200_dist_seg_f64' in tb_double.CALLS
    assert_same_samples(lock, serial)


def _fallback_models():
    m = exma2.get_model(seed_obs=4)
    elfi.AdaptiveDistance(m['S1'], m['S2'], name='ad')
    elfi.Distance(lambda X, Y: ssd.cdist(X.cpu().numpy(), Y), m['S1'], m['S2'], name='dc')
    elfi.Distance('euclidean', m['S1'], m['S2'], w=[1.0, 2.0], name='dw')
    return m


@pytest.mark.parametrize('case', ['threshold', 'adaptive', 'pool', 'callable', 'weighted', 'smc'])
def test_fallback_runs_serially(tb_double, case):
    m = _fallback_models()
    mk = dict(discrepancy_name='d', batch_size=100)
    sk = dict(n_samples=20, quantile=0.1)
    method = None
    if case == 'threshold':
        sk = dict(n_samples=20, threshold=0.5)
    elif case == 'adaptive':
        mk['discrepancy_name'] = 'ad'
    elif case == 'pool':
        mk['pool'] = elfi.OutputPool(['S1', 'S2'])
    elif case == 'callable':
        mk['discrepancy_name'] = 'dc'
    elif case == 'weighted':
        mk['discrepancy_name'] = 'dw'
    elif case == 'smc':
        method = elfi.SMC
        sk = dict(n_samples=20, thresholds=[2.0, 1.0])
    tb = elfi.Testbench(model=m, repetitions=2, seed=3, progress_bar=False)
    tm = elfi.TestbenchMethod(method=method or elfi.Rejection)
    tm.set_method_kwargs(**mk)
    assert tb._lockstep_metric(tm) is None or case == 'threshold'
    tm.set_sample_kwargs(bar=False, **sk)
    assert tb._lockstep_metric(tm) is None
    if case == 'pool':      # a pool pins one seed: only a single inference can use it
        return
    tb.add_method(tm)
    tb.run()
    assert not set(SEG) & set(tb_double.CALLS)
    assert len(tb.testbench_results[0]['results']) == 2
