"""TwoStageSelection host logic on the CPU double of the C ABI: the API, the reference's fixtures on
the host MA2 model, and the all-combination path against the per-combination loop."""
import logging
from functools import partial

import numpy as np
import pytest

import abi_double
import diagnostics_double
from conftest import load_golden
from elfi_b200 import TwoStageSelection, diagnostics
from elfi_b200 import model as em
from elfi_b200.examples import gauss, ma2


def ac_round(x, lag):
    """The autocovariance rounded to one decimal (host data)."""
    return np.round(np.mean(x[:, lag:] * x[:, :-lag], axis=1), 1)


def named(fn, name, **kw):
    f = partial(fn, **kw)
    f.__name__ = name
    return f


AC1 = named(ma2.autocov, 'ac_lag1', lag=1)
AC2 = named(ma2.autocov, 'ac_lag2', lag=2)
R1 = named(ac_round, 'ac_round1', lag=1)
R2 = named(ac_round, 'ac_round2', lag=2)

# the cases of tests/golden/gen_golden_diagnostics.py
CASES = {'ma2': (dict(list_ss=[AC1, AC2, gauss.ss_mean]), False),
         'twice': (dict(prepared_ss=[(AC1,), (AC1, AC2), (AC1,)]), False),
         'round': (dict(list_ss=[R1, R2]), False),
         'dup': (dict(list_ss=[AC1, AC2]), True)}


def simulator(discrete=False, fn=ma2.MA2):
    """The reference's unit-test MA2 model on the host (observed data from RandomState(0))."""
    m = em.ElfiModel()
    if discrete:
        t1 = em.Prior('randint', -1, 2, model=m, name='t1')
        t2 = em.Prior('randint', 0, 2, model=m, name='t2')
    else:
        t1 = em.Prior(ma2.CustomPrior1, 2, model=m, name='t1')
        t2 = em.Prior(ma2.CustomPrior2, t1, 1, name='t2')
    y_obs = ma2.MA2(.6, .2, random_state=np.random.RandomState(0))
    return em.Simulator(fn, t1, t2, observed=y_obs, name='MA2')


def case(name):
    g = load_golden('diagnostics')
    kw, discrete = CASES[name]
    n_sim, batch_size, seed, n_acc, n_closest = (int(v) for v in g[name + '_config'])
    sel = TwoStageSelection(simulator(discrete), 'euclidean', seed=seed, **kw)
    return g, sel, dict(n_sim=n_sim, n_acc=n_acc, n_closest=n_closest, batch_size=batch_size)


def close(a, b, tol=1e-10):
    a, b = np.asarray(a, dtype=float), np.asarray(b, dtype=float)
    same_inf = np.isinf(a) & (a == b)
    with np.errstate(invalid='ignore'):
        return np.all(same_inf | (np.abs(a - b) <= tol * (1 + np.abs(b))))


@pytest.fixture
def double(cpu_double, monkeypatch):
    abi_double.install(monkeypatch, diagnostics_double.TABLE)
    return cpu_double


def test_errors_and_defaults(double):
    with pytest.raises(ValueError, match='No summary statistics to assess.'):
        TwoStageSelection(simulator(), 'euclidean')
    sel = TwoStageSelection(simulator(), 'euclidean', list_ss=[AC1])
    for kw in (dict(n_sim=199), dict(n_sim=1000, n_acc=2000), dict(n_sim=1000, n_acc=10,
                                                                      n_closest=11)):
        with pytest.raises(ValueError, match='The number of simulations is too small.'):
            sel.run(**kw)


def test_combination_order_and_clamp():
    sel = TwoStageSelection(simulator(), 'euclidean', list_ss=[AC1, AC2, R1], max_cardinality=9)
    assert sel.ss_candidates == [(AC1,), (AC2,), (R1,), (AC1, AC2), (AC1, R1), (AC2, R1),
                                 (AC1, AC2, R1)]
    sel = TwoStageSelection(simulator(), 'euclidean', list_ss=[AC1, AC2, R1], max_cardinality=1)
    assert sel.ss_candidates == [(AC1,), (AC2,), (R1,)]


def test_prepared_ss_as_lists(double):
    sel = TwoStageSelection(simulator(), 'euclidean', prepared_ss=[[AC1], [AC1, AC2]], seed=1)
    assert sel.ss_candidates == [(AC1,), (AC1, AC2)]
    assert sel.run(2000, n_acc=100, n_closest=5, batch_size=500) in sel.ss_candidates


@pytest.mark.parametrize('name', ['dup', 'ma2', 'twice'])
def test_golden_on_host_model(double, name, caplog):
    g, sel, kw = case(name)
    thetas = sel._device_accepted_thetas(kw['n_sim'], kw['n_acc'], kw['batch_size'])
    assert np.array_equal(thetas.cpu().numpy(), g[name + '_thetas'])
    with caplog.at_level(logging.INFO, logger='elfi_b200.diagnostics'):
        chosen = sel.run(**kw)
    assert chosen == sel.ss_candidates[int(g[name + '_selected'])]
    assert close([s['entropy'] for s in sel.scores], g[name + '_entropy'])
    assert close([s['mrsse'] for s in sel.scores], g[name + '_mrsse'])
    assert [s['names'] for s in sel.scores] == [[f.__name__ for f in c] for c in sel.ss_candidates]
    assert sum('shows the entropy of' in r.message for r in caplog.records) == len(sel.scores)
    assert sum('The minimum MRSSE' in r.message for r in caplog.records) == 1


def test_golden_with_tied_distances(double):
    """Rounded summaries tie.  The reference's merge sorts with NumPy's unstable quicksort, so
    among tied rows it keeps other rows in another order than this repository's stable Rejection;
    the device path follows Rejection, and the selection is the reference's."""
    g, sel, kw = case('round')
    thetas = sel._device_accepted_thetas(kw['n_sim'], kw['n_acc'], kw['batch_size']).cpu().numpy()
    for c, set_ss in enumerate(sel.ss_candidates):
        loop = sel._obtain_accepted_thetas(set_ss, kw['n_sim'], kw['n_acc'], kw['batch_size'])
        assert np.array_equal(thetas[c], loop.cpu().numpy())
    assert sel.run(**kw) == sel.ss_candidates[int(g['round_selected'])]


@pytest.mark.parametrize('metric', diagnostics.DEVICE_METRICS)
def test_device_path_equals_loop(double, metric, monkeypatch):
    """One combination at a time in chunks of 700 rows, which cut across the 500-row batches: the
    kept rows still follow one stable order by (distance, row), which is what the batch-by-batch
    merge of Rejection keeps."""
    sel = TwoStageSelection(simulator(), metric, list_ss=[AC1, AC2, R1], seed=3)
    monkeypatch.setattr(diagnostics, 'DISTANCE_BLOCK_BYTES', 8 * 700)
    dev_thetas = sel._device_accepted_thetas(3000, 60, 500).cpu().numpy()
    for c, set_ss in enumerate(sel.ss_candidates):
        loop = sel._obtain_accepted_thetas(set_ss, 3000, 60, 500).cpu().numpy()
        assert np.array_equal(dev_thetas[c], loop), set_ss


def test_callable_distance_takes_the_loop(double):
    def host(v):
        return np.asarray(v.cpu()) if hasattr(v, 'cpu') else np.asarray(v)

    def euclid(*simulated, observed):
        X = np.column_stack([host(s) for s in simulated])
        return np.sqrt(np.sum((X - np.column_stack([host(o) for o in observed])) ** 2, axis=1))
    ref = TwoStageSelection(simulator(), 'euclidean', list_ss=[AC1, AC2], seed=2)
    sel = TwoStageSelection(simulator(), euclid, list_ss=[AC1, AC2], seed=2)
    del double.CALLS[:]
    assert sel.run(2000, n_acc=50, n_closest=5, batch_size=500) == \
        ref.run(2000, n_acc=50, n_closest=5, batch_size=500)
    assert [s['names'] for s in sel.scores] == [s['names'] for s in ref.scores]


def test_device_path_simulates_each_batch_once(double):
    calls = []

    def counted(*args, **kw):
        calls.append(kw['batch_size'])
        return ma2.MA2(*args, **kw)
    sel = TwoStageSelection(simulator(fn=counted), 'euclidean', list_ss=[AC1, AC2, R1], seed=0)
    sel.run(2500, n_acc=50, n_closest=5, batch_size=1000)
    assert calls == [1000] * 3
    assert len(sel.scores) == 7


def test_multi_rank_error(double, monkeypatch):
    class TwoRanks:
        on = True
    monkeypatch.setattr(diagnostics, 'Comm', TwoRanks)
    sel = TwoStageSelection(simulator(), 'euclidean', list_ss=[AC1])
    with pytest.raises(RuntimeError, match='one rank'):
        sel.run(2000, n_acc=50, n_closest=5, batch_size=500)


def test_scoring_kernels_on_crafted_sets(double):
    """ops.knn_entropy / ops.mrsse (through the double) against the reference's _calc_entropy and
    _calc_MRSSE on the crafted point sets of the fixture."""
    from elfi_b200 import ops
    g = load_golden('diagnostics')
    off = 0
    for (q, k, n, m), E, M in zip(g['pts_config'], g['pts_entropy'], g['pts_mrsse']):
        X = g['pts_data'][off:off + n * q].reshape(n, q)
        off += n * q
        _, logsum = ops.knn_entropy(X, k)
        e = TwoStageSelection._entropy(q, n, k, logsum.cpu().numpy()[0])
        assert close(e, E), (q, k, n)
        assert close(ops.mrsse(X, X[:m]).cpu().numpy()[0], M), (q, k, n)
