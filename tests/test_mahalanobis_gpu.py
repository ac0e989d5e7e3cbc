"""elfi_b200_dist_mahalanobis_thr_f64 on the device: ops.dist_mahalanobis bit for bit against
SciPy's cdist(..., 'mahalanobis', VI=VI), its acceptance outputs, Distance nodes in the host and the
device MA2 model, and the reference's MA2 runs (tests/golden/gen_golden_mahalanobis.py)."""
import numpy as np
import pytest
import torch
from scipy.spatial.distance import cdist

import mahalanobis_cases as cases

pytestmark = pytest.mark.gpu

ROWS = (0, 1, 37, 100003)


def _check(S, obs, VI, thr):
    """S: host rows, or a device view whose rows are further apart than D (ldS > D)."""
    from elfi_b200 import ops
    host = S.cpu().numpy() if hasattr(S, 'cpu') else S
    ref = cdist(host, obs[None], 'mahalanobis', VI=VI).ravel() if len(S) else np.empty(0)
    d, idx = ops.dist_mahalanobis(S, obs, VI, threshold=thr)
    d, idx = d.cpu().numpy(), idx.cpu().numpy()
    assert cases.same_bits(d, ref)
    assert np.array_equal(idx, np.nonzero(ref <= thr)[0])
    return ref


@pytest.mark.parametrize('kind', cases.KINDS)
@pytest.mark.parametrize('D', cases.DIMS)
def test_matches_cdist(D, kind):
    """Every B, contiguous rows and rows inside a wider matrix (ldS > D), NaN and +-inf rows."""
    rs = np.random.RandomState(100 + D * 3 + cases.KINDS.index(kind))
    VI = cases.make_vi(kind, D, rs)
    obs = rs.randn(D)
    for B in ROWS:
        if B == 100003 and kind != 'symmetric' and D > 64:
            continue    # cdist's time, not the kernel's: the wide B runs every D once, symmetric
        S = cases.make_rows(B, D, rs, obs)
        ref = _check(S, obs, VI, 1.0)
        wide = np.full((B, D + 5), np.nan)
        wide[:, 2:2 + D] = S
        view = torch.from_numpy(wide).cuda()[:, 2:2 + D]
        assert B < 2 or view.stride(0) == D + 5
        _check(view, obs, VI, float(np.nanmedian(ref)) if B > 5 else 1.0)


def test_thresholds_and_counts():
    from elfi_b200 import ops
    rs = np.random.RandomState(5)
    D = 16
    VI, obs = cases.make_vi('nonsymmetric', D, rs), rs.randn(D)
    S = cases.make_rows(20000, D, rs, obs)
    ref = cdist(S, obs[None], 'mahalanobis', VI=VI).ravel()
    for thr in (-1.0, 0.0, float(ref[7]), float(np.nanquantile(ref, 0.3)), np.inf, np.nan):
        d, idx = ops.dist_mahalanobis(S, obs, VI, threshold=thr)
        assert np.array_equal(idx.cpu().numpy(), np.nonzero(ref <= thr)[0]), thr
        _, n = ops.dist_mahalanobis(S, obs, VI, threshold=thr, want_indices=False)
        assert n == np.count_nonzero(ref <= thr), thr
    d, idx = ops.dist_mahalanobis(S, obs, VI)
    assert idx is None and cases.same_bits(d.cpu().numpy(), ref)


def test_repeated_calls_are_identical():
    from elfi_b200 import ops
    rs = np.random.RandomState(9)
    D = 145
    VI, obs = cases.make_vi('symmetric', D, rs), rs.randn(D)
    S = cases.make_rows(50001, D, rs, obs)
    first = ops.dist_mahalanobis(S, obs, VI)[0].cpu().numpy()
    for _ in range(3):
        assert cases.same_bits(ops.dist_mahalanobis(S, obs, VI)[0].cpu().numpy(), first)


def test_argument_errors():
    from elfi_b200 import ops
    D = cases.D_MAX + 1
    with pytest.raises(ValueError, match='MAHALANOBIS_D_MAX'):
        ops.dist_mahalanobis(np.ones((3, D)), np.zeros(D), np.eye(D))
    with pytest.raises(ValueError, match='VI must be a'):
        ops.dist_mahalanobis(np.ones((3, 4)), np.zeros(4), np.eye(5))


def test_node_in_a_model():
    cases.case_node_in_a_model()


def test_pilot_matches_reference():
    cases.case_pilot()


@pytest.mark.parametrize('run', cases.RUNS)
def test_rejection_matches_reference(run):
    cases.case_rejection(run)


def test_smc_matches_reference():
    cases.case_smc()


def test_rejection_on_the_device_model():
    """A Mahalanobis node on the device MA2 model: the accepted distances are cdist of the
    materialised summaries."""
    import elfi_b200 as elfi
    from elfi_b200 import device as dev
    from elfi_b200.examples import ma2
    g = cases.load_golden('ma2_mahalanobis')
    m = ma2.get_device_model(seed_obs=4)
    node = elfi.Distance('mahalanobis', m['S1'], m['S2'], VI=g['VI'], name='dm')
    res = elfi.Rejection(node, batch_size=10000, seed=3, output_names=['S1', 'S2']).sample(
        200, quantile=0.01, bar=False)
    S = np.column_stack([np.asarray(res.outputs[k], dtype=np.float64).ravel()
                         for k in ('S1', 'S2')])
    obs = np.array([float(dev.to_host(m[k].observed).ravel()[0]) for k in ('S1', 'S2')])
    assert res.n_samples == 200 and res.n_sim == 20000
    assert cases.same_bits(res.discrepancies, cdist(S, obs[None], 'mahalanobis', VI=g['VI']).ravel())
