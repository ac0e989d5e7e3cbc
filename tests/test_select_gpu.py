"""GPU parity: sort / gather / weighted quantile / top-n merge vs NumPy and reference goldens."""
import numpy as np
import pytest

import elfi_oracle as o
from conftest import load_golden

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('n', [1, 2, 31, 32, 33, 1000, 1024, 1025, 5000, 100000, 1_000_003])
def test_argsort_matches_numpy(n):
    from elfi_b200 import ops
    rs = np.random.RandomState(n)
    x = np.abs(rs.randn(n)) * 10 ** rs.uniform(-3, 3, n)
    perm, ks = ops.argsort(x, return_keys=True)
    ref = np.argsort(x, kind='stable')
    assert np.array_equal(perm.cpu().numpy(), ref)
    assert np.array_equal(ks.cpu().numpy(), x[ref])


def test_argsort_special_values_and_stability():
    from elfi_b200 import ops
    x = np.array([3.0, np.inf, 0.0, -0.0, 1.5, np.nan, -2.0, 1.5, np.inf, 1.5, -np.inf, 5e-324])
    perm = ops.argsort(x).cpu().numpy()
    xs = x[perm]
    assert np.isnan(xs[-1])
    assert np.array_equal(xs[:-1], np.sort(x)[:-1])
    ties = [i for i in perm if x[i] == 1.5]
    assert ties == sorted(ties)                      # stable
    x = np.repeat(np.arange(50.0), 400)[np.random.RandomState(0).permutation(20000)]
    assert np.array_equal(ops.argsort(x).cpu().numpy(), np.argsort(x, kind='stable'))


def test_take_rows():
    from elfi_b200 import ops
    rs = np.random.RandomState(1)
    a = rs.randn(1000, 7)
    idx = rs.randint(0, 1000, 333).astype(np.int32)
    assert np.array_equal(ops.take_rows(a, idx).cpu().numpy(), a[idx])
    v = rs.randn(1000)
    assert np.array_equal(ops.take_rows(v, idx).cpu().numpy(), v[idx])
    t3 = rs.randn(100, 3, 2)
    assert np.array_equal(ops.take_rows(t3, idx[:50] % 100).cpu().numpy(), t3[idx[:50] % 100])


def test_weighted_quantile_golden():
    from elfi_b200 import ops
    g = load_golden('weighted_quantile')
    for a, qw, qu in zip(g['alphas'], g['q_w'], g['q_unw']):
        assert ops.weighted_sample_quantile(g['x'], a, g['w']) == qw
        assert ops.weighted_sample_quantile(g['x'], a) == qu


@pytest.mark.parametrize('n', [2, 10, 200, 1000, 5000, 100000])
def test_weighted_quantile_equal_weights_knife_edge(n):
    """alpha exactly on a cumulative weight: the sequential rounding decides (SMC round 0)."""
    from elfi_b200 import ops
    rs = np.random.RandomState(n)
    x = rs.rand(n)
    for a in (0.1, 0.2, 0.25, 0.3, 0.5, 0.7, 0.75, 0.9):
        assert ops.weighted_sample_quantile(x, a) == o.weighted_sample_quantile(x, a)
        assert ops.weighted_sample_quantile(x, a, np.ones(n)) == o.weighted_sample_quantile(
            x, a, np.ones(n))
        w3 = np.full(n, 3.0)
        assert ops.weighted_sample_quantile(x, a, w3) == o.weighted_sample_quantile(x, a, w3)


@pytest.mark.parametrize('n', [1, 2, 100, 4096, 4097, 250000, 1000003])
def test_weighted_quantile_vs_oracle(n):
    from elfi_b200 import ops
    rs = np.random.RandomState(n)
    x = rs.rand(n)
    w = rs.rand(n) ** 3
    for a in (0.0, 0.05, 0.3333, 0.5, 0.99, 1.0):
        assert ops.weighted_sample_quantile(x, a, w) == o.weighted_sample_quantile(x, a, w)


@pytest.mark.parametrize('B,n', [(1000, 256), (37, 1), (500, 2), (333, 50), (100, 257), (64, 1000),
                                 (9, 2048), (77, 31), (77, 32), (77, 33), (300, 64), (41, 100),
                                 (129, 127), (50, 511), (50, 512), (50, 513), (3001, 255)])
def test_rowsort_matches_numpy(B, n):
    from elfi_b200 import ops
    rs = np.random.RandomState(B + n)
    x = rs.randn(B, n) * 10 ** rs.uniform(-2, 2, (B, 1))
    if n >= 8:
        x[::5, 3] = np.nan
        x[::7, 1] = np.inf
        x[::11, 0] = -np.inf
        x[::3, 2] = x[::3, 4]                 # ties
    got = ops.rowsort(x).cpu().numpy()
    assert np.array_equal(got, np.sort(x, axis=1), equal_nan=True)
    if n >= 4:                                # strided rows, odd offset: the unaligned load path
        from elfi_b200 import device as dev
        got = ops.rowsort(dev.to_device(x)[:, 1:n - 1]).cpu().numpy()
        assert np.array_equal(got, np.sort(x[:, 1:n - 1], axis=1), equal_nan=True)


def test_rowsort_rejects_too_wide_rows_without_poisoning_the_context():
    from elfi_b200 import _lib, ops
    with pytest.raises(_lib.ElfiB200Error):
        ops.rowsort(np.zeros((4, 4096)))
    assert np.array_equal(ops.rowsort(np.array([[3.0, 1.0, 2.0]])).cpu().numpy(), [[1.0, 2.0, 3.0]])
