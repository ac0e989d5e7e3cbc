"""GPU parity: CUDA distance + acceptance (through the C ABI) vs the CPU oracle, bit-exact."""
import numpy as np
import pytest

import elfi_oracle as o
from conftest import load_golden

pytestmark = pytest.mark.gpu


def _check(B, D, K=1, weighted=False, q=0.05, ld=None, seed=0):
    import torch
    from elfi_b200 import ops
    rs = np.random.RandomState(seed)
    S_full = rs.randn(B, ld or D)
    S = S_full[:, :D]
    obs = rs.randn(1, D)
    if weighted or K > 1:
        ws = [None if (k == 0 and not weighted) else rs.rand(D) + 0.2 for k in range(K)]
        ref = o.nested_distance(S, obs, ws)
        W = np.stack([np.ones(D) if w is None else w ** 2 for w in ws])
    else:
        ref = o.cdist_euclid(S, obs)[:, None]
        W = None
    thr = np.quantile(ref, q, axis=0) if B > 0 else np.zeros(K)
    ref_idx = o.accept_indices(ref, thr)
    St = torch.from_numpy(S_full).cuda()[:, :D]
    d, idx = ops.dist_euclid(St, obs, w=W, thresholds=thr)
    d = d.cpu().numpy().reshape(B, K)
    idx = idx.cpu().numpy()
    assert np.array_equal(d, ref), 'distances differ from the oracle'
    assert np.array_equal(idx, ref_idx), 'accepted index set differs'
    return len(idx)


@pytest.mark.parametrize('B,D', [(4096, 128), (1000, 128), (33, 16), (31, 130), (5000, 17),
                                 (1, 128), (100000, 128), (2049, 256), (777, 48), (64, 1000)])
def test_euclid_tma_path(B, D):
    _check(B, D, seed=B + D)


@pytest.mark.parametrize('B,D', [(1000, 2), (999, 1), (50000, 2), (33, 7), (4097, 15)])
def test_euclid_direct_path(B, D):
    _check(B, D, seed=B * 3 + D)


def test_euclid_strided_rows():
    _check(3000, 128, ld=160, seed=5)      # TMA with ld != D
    _check(3000, 21, ld=33, seed=6)        # odd ld -> direct path


def test_empty_batch():
    from elfi_b200 import ops
    d, idx = ops.dist_euclid(np.zeros((0, 8)), np.zeros(8), thresholds=1.0)
    assert d.shape[0] == 0 and idx.shape[0] == 0


@pytest.mark.parametrize('K', [1, 2, 3, 5, 8, 13, 32])
def test_nested_weighted(K):
    _check(3000, 256, K=K, weighted=(K == 1), q=0.6, seed=K)
    _check(1500, 6, K=K, weighted=(K == 1), q=0.6, seed=K + 100)


def test_weights_of_ones_equal_unweighted():
    import torch
    from elfi_b200 import ops
    rs = np.random.RandomState(9)
    S = rs.randn(2000, 64)
    obs = rs.randn(64)
    d0, _ = ops.dist_euclid(S, obs)
    d1, _ = ops.dist_euclid(S, obs, w=np.ones(64))
    assert torch.equal(d0, d1)


def test_accept_all_and_none():
    from elfi_b200 import ops
    rs = np.random.RandomState(1)
    S = rs.randn(5000, 32)
    obs = rs.randn(32)
    _, idx = ops.dist_euclid(S, obs, thresholds=np.inf)
    assert np.array_equal(idx.cpu().numpy(), np.arange(5000))
    _, idx = ops.dist_euclid(S, obs, thresholds=-1.0)
    assert idx.numel() == 0


def test_nan_rows_are_rejected():
    from elfi_b200 import ops
    rs = np.random.RandomState(2)
    S = rs.randn(1000, 32)
    S[::7, 3] = np.nan
    obs = rs.randn(32)
    d, idx = ops.dist_euclid(S, obs, thresholds=1e9)
    ref = o.cdist_euclid(S, obs)
    assert np.array_equal(d.cpu().numpy(), ref, equal_nan=True)
    assert np.array_equal(idx.cpu().numpy(), o.accept_indices(ref, 1e9))


def test_golden_ma2_distance():
    from elfi_b200 import ops
    g = load_golden('ma2_generate')
    S = np.column_stack([g['S1'], g['S2']])
    obs = np.array([g['obs_S1'][0], g['obs_S2'][0]])
    d, _ = ops.dist_euclid(S, obs)
    assert np.array_equal(d.cpu().numpy(), g['d'])


def test_full_size_config2_properties():
    """BASELINE config #2 shape (1e6 x 128): sampled rows bit-exact vs the oracle, accepted set
    consistent with the distances, count equals a direct count."""
    import torch
    from elfi_b200 import ops
    B, D = 1_000_000, 128
    gen = torch.Generator(device='cuda').manual_seed(0)
    S = torch.randn(B, D, dtype=torch.float64, device='cuda', generator=gen)
    obs = torch.randn(D, dtype=torch.float64, device='cuda', generator=gen)
    d, _ = ops.dist_euclid(S, obs)
    thr = float(torch.quantile(d[:100000], 0.01))
    d2, idx = ops.dist_euclid(S, obs, thresholds=thr)
    assert torch.equal(d, d2)
    assert torch.equal(idx.long(), torch.nonzero(d <= thr).ravel())
    rows = torch.cat([torch.arange(0, 2048), torch.arange(B - 2048, B),
                      torch.randint(0, B, (4096,))]).cuda()
    ref = o.cdist_euclid(S[rows].cpu().numpy(), obs.cpu().numpy())
    assert np.array_equal(d[rows].cpu().numpy(), ref)
