"""TwoStageSelection on the device: the three entry points against SciPy, the all-combination path
against Rejection, the reference's fixtures and its own unit-test assertion."""
from functools import partial

import numpy as np
import pytest
import torch

import diagnostics_double as dd
from elfi_b200 import TwoStageSelection, diagnostics, ops
from elfi_b200 import device as dev
from elfi_b200.examples import gauss, ma2
from elfi_b200.throughput import LazySimulation
from test_diagnostics_host import AC1, AC2, R1, case, close, named, simulator

pytestmark = pytest.mark.gpu


def random_layout(rs, widths, n_comb):
    starts = np.concatenate([[0], np.cumsum(widths)[:-1]])
    combs = []
    for _ in range(n_comb):
        pick = rs.choice(len(widths), size=rs.randint(1, min(6, len(widths)) + 1), replace=False)
        combs.append([(int(starts[j]), int(widths[j])) for j in pick])
    return combs


@pytest.mark.parametrize('metric', diagnostics.DEVICE_METRICS)
def test_subset_distance_bit_exact(metric):
    rs = np.random.RandomState(11)
    widths = rs.randint(1, 9, size=9)
    W = int(widths.sum())
    combs = random_layout(rs, widths, 60)
    B = 3001
    full = rs.randn(B, W + 5)
    full[7, 3] = np.nan
    full[8, :] = np.inf
    full[9, 1] = -np.inf
    full[10, 0], full[10, 2] = np.inf, np.nan
    S = full[:, 2:2 + W]                      # a strided view
    obs = rs.randn(W)
    layout = ops.SubsetLayout(combs, W)
    Sd = dev.to_device(full)[:, 2:2 + W]
    got = ops.subset_distance(Sd, obs, layout, metric).cpu().numpy()
    want = dd.subset_distance(S, obs, combs, metric)
    assert np.array_equal(got, want, equal_nan=True)
    again = ops.subset_distance(Sd, obs, layout, metric).cpu().numpy()
    assert np.array_equal(got, again, equal_nan=True)


def test_subset_distance_errors():
    with pytest.raises(ValueError):
        ops.SubsetLayout([[(0, 3)]], 2)
    with pytest.raises(ValueError):
        ops.SubsetLayout([[(0, 1)]], 513)
    layout = ops.SubsetLayout([[(0, 1)]], 2)
    with pytest.raises(ValueError):
        ops.subset_distance(np.zeros((4, 2)), np.zeros(2), layout, 'minkowski')


def nan_ac1(x):
    """ac_lag1 with every 97th row NaN and every 89th +inf."""
    v = ma2.autocov(x, 1).clone()
    v[::97] = float('nan')
    v[3::89] = float('inf')
    return v


@pytest.mark.parametrize('metric', diagnostics.DEVICE_METRICS)
def test_selection_equals_rejection(metric, monkeypatch):
    ac_nan = named(nan_ac1, 'ac_nan')
    sel = TwoStageSelection(simulator(), metric, list_ss=[AC1, R1, ac_nan], seed=5)
    monkeypatch.setattr(diagnostics, 'DISTANCE_BLOCK_BYTES', 8 * 1300)
    thetas = sel._device_accepted_thetas(6000, 400, 1000).cpu().numpy()
    for c, set_ss in enumerate(sel.ss_candidates):
        loop = sel._obtain_accepted_thetas(set_ss, 6000, 400, 1000).cpu().numpy()
        assert np.array_equal(thetas[c], loop), set_ss


@pytest.mark.parametrize('q', [1, 2, 5, 16])
@pytest.mark.parametrize('k', [1, 4, 7, 32])
def test_knn_radii_against_ckdtree(q, k):
    rs = np.random.RandomState(q * 100 + k)
    for n in sorted({k, k + 1, 300, 2000 if q < 16 else 700}):
        X = rs.randn(3, n, q)
        R, logsum = ops.knn_entropy(X, k)
        R, logsum = R.cpu().numpy(), logsum.cpu().numpy()
        for c in range(3):
            want = dd.knn_radii(X[c], k)
            assert np.all(np.abs(R[c] - want) <= 1e-12 * np.abs(want)), (q, k, n)
            e = TwoStageSelection._entropy(q, n, k, logsum[c])
            e_ref = TwoStageSelection._entropy(q, n, k, np.sum(np.log(want)))
            assert close(e, e_ref), (q, k, n)
        R2, logsum2 = ops.knn_entropy(X, k)
        assert np.array_equal(R, R2.cpu().numpy()) and np.array_equal(logsum, logsum2.cpu().numpy())


def test_knn_duplicates_and_short_sets():
    rs = np.random.RandomState(3)
    X = rs.randn(50, 3)
    X[10:14] = X[9]
    R, logsum = ops.knn_entropy(X, 4)
    assert np.all(R.cpu().numpy()[9:14] == 0) and logsum.cpu().numpy()[0] == -np.inf
    R, logsum = ops.knn_entropy(X[:5], 8)
    assert np.all(R.cpu().numpy() == np.inf) and logsum.cpu().numpy()[0] == np.inf
    with pytest.raises(ValueError):
        ops.knn_entropy(X, 33)
    with pytest.raises(ValueError):
        ops.knn_entropy(rs.randn(10, 17), 2)


def test_knn_large_set():
    rs = np.random.RandomState(4)
    X = rs.randn(20000, 2)
    R, _ = ops.knn_entropy(X, 4)
    want = dd.knn_radii(X, 4)
    assert np.all(np.abs(R.cpu().numpy()[0] - want) <= 1e-12 * want)


def test_mrsse_against_reference():
    rs = np.random.RandomState(5)
    T = rs.randn(4, 500, 3)
    P = rs.randn(20, 3)
    got = ops.mrsse(T, P).cpu().numpy()
    assert close(got, [dd.mrsse(T[c], P) for c in range(4)])
    assert np.array_equal(got, ops.mrsse(T, P).cpu().numpy())


@pytest.mark.parametrize('name', ['dup', 'ma2', 'twice'])
def test_golden_on_device(name):
    g, sel, kw = case(name)
    thetas = sel._device_accepted_thetas(kw['n_sim'], kw['n_acc'], kw['batch_size'])
    assert np.array_equal(thetas.cpu().numpy(), g[name + '_thetas'])
    assert sel.run(**kw) == sel.ss_candidates[int(g[name + '_selected'])]
    assert close([s['entropy'] for s in sel.scores], g[name + '_entropy'])
    assert close([s['mrsse'] for s in sel.scores], g[name + '_mrsse'])


def materialised(stat):
    """A summary of the simulated data itself: lazy simulator output is materialised first, since
    gauss.ss_mean on a LazySimulation would return the fused lag-1 autocovariance."""
    def fn(y):
        return stat(y.materialize() if isinstance(y, LazySimulation) else y)
    return fn


def test_reference_assertion_on_device_model():
    mean = named(materialised(gauss.ss_mean), 'ss_mean')
    m = ma2.get_device_model(seed_obs=0)
    sel = TwoStageSelection(m['MA2'], 'euclidean', list_ss=[AC1, AC2, mean], seed=0)
    chosen = sel.run(n_sim=100000, batch_size=10000)
    assert AC1 in chosen and AC2 in chosen and mean not in chosen


def test_large_run_on_device_model():
    lags = [named(materialised(partial(ma2.autocov, lag=lag)), 'ac{}'.format(lag))
            for lag in range(1, 9)]
    cands = lags + [named(materialised(gauss.ss_mean), 'mean'),
                    named(materialised(gauss.ss_var), 'var')]
    m = ma2.get_device_model(seed_obs=0)
    sel = TwoStageSelection(m['MA2'], 'euclidean', list_ss=cands, max_cardinality=3, seed=0)
    assert len(sel.ss_candidates) == 175
    sel.run(n_sim=10 ** 6, batch_size=10 ** 5)
    thetas = sel._device_accepted_thetas(10 ** 6, 10 ** 4, 10 ** 5)
    for c in (0, 57, 174):
        loop = sel._obtain_accepted_thetas(sel.ss_candidates[c], 10 ** 6, 10 ** 4, 10 ** 5)
        assert torch.equal(thetas[c], loop)
