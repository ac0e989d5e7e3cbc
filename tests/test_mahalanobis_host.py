"""The Mahalanobis distance's order of operations against SciPy, and ops.dist_mahalanobis's argument
checks, without a GPU.

tests/mahalanobis_double.py replays the order that elfi_b200_dist_mahalanobis_thr_f64 follows
(t = VI u by ROWS of VI and then u . t, each in SciPy's even/odd two-sum order, every operation
rounded on its own).  Here the replay is held to cdist bit for bit, and two near misses are shown to
differ from it, so the checks can tell the order apart."""
import numpy as np
import pytest
from scipy.spatial.distance import cdist

import abi_double
import mahalanobis_cases as cases
import mahalanobis_double as md


@pytest.mark.parametrize('kind', cases.KINDS)
@pytest.mark.parametrize('D', cases.DIMS)
def test_replay_matches_cdist(D, kind):
    rs = np.random.RandomState(D * 3 + cases.KINDS.index(kind))
    VI = cases.make_vi(kind, D, rs)
    obs = rs.randn(D)
    S = cases.make_rows(300, D, rs, obs)
    ref = cdist(S, obs[None], 'mahalanobis', VI=VI).ravel()
    assert cases.same_bits(md.cdist_mahalanobis(S, obs, VI), ref)
    assert np.isnan(ref[0]) and not np.isfinite(ref[:3]).any()   # NaN and +-inf rows
    if kind != 'indefinite':
        assert np.isfinite(ref[5:]).all()
    else:
        assert np.isnan(ref[5:]).any() and (D == 1 or np.isfinite(ref[5:]).any())


def _one_sum(terms):
    s = np.zeros(terms.shape[:-1])
    for j in range(terms.shape[-1]):
        s = s + terms[..., j]
    return s


def test_order_is_discriminating():
    """Columns of VI instead of rows, or one running sum instead of two, give other bits."""
    rs = np.random.RandomState(3)
    D = 33
    VI = cases.make_vi('nonsymmetric', D, rs)
    obs = rs.randn(D)
    S = cases.make_rows(400, D, rs, obs)[5:]
    ref = cdist(S, obs[None], 'mahalanobis', VI=VI).ravel()
    assert not cases.same_bits(md.cdist_mahalanobis(S, obs, VI.T), ref)
    u = S - obs
    one = np.sqrt(_one_sum(u * _one_sum(VI[None] * u[:, None, :])))
    assert not cases.same_bits(one, ref)


def test_limit_is_the_header_constant():
    from elfi_b200 import _lib, ops
    assert ops.MAHALANOBIS_D_MAX == _lib.CONSTANTS['MAHALANOBIS_D_MAX'] == md.D_MAX == cases.D_MAX
    assert md.D_MAX >= _lib.CONSTANTS['SYNLIK_D_MAX']
    assert 'mahalanobis' not in ops.METRIC_CODES and 'mahalanobis' not in ops.SUBSET_METRIC_CODES
    assert 'mahalanobis' not in ops.SEG_METRICS


@pytest.fixture
def double(cpu_double, monkeypatch):
    abi_double.install(monkeypatch, md.TABLE)
    return cpu_double


def test_operator_on_the_double(double):
    from elfi_b200 import ops
    rs = np.random.RandomState(1)
    VI = cases.make_vi('nonsymmetric', 5, rs)
    obs = rs.randn(5)
    S = cases.make_rows(50, 5, rs, obs)
    ref = cdist(S, obs[None], 'mahalanobis', VI=VI).ravel()
    d, idx = ops.dist_mahalanobis(S, obs, VI, threshold=1.5)
    assert cases.same_bits(d.cpu().numpy(), ref)
    assert np.array_equal(idx.cpu().numpy(), np.nonzero(ref <= 1.5)[0])
    d, n = ops.dist_mahalanobis(S, obs, VI, threshold=1.5, want_indices=False)
    assert n == np.count_nonzero(ref <= 1.5)
    d, idx = ops.dist_mahalanobis(S[:0], obs, VI, threshold=1.5)
    assert d.shape == (0,) and len(idx) == 0


@pytest.mark.parametrize('shape', [(5,), (4, 5), (5, 4), (6, 6), (1, 5, 5)])
def test_vi_of_the_wrong_shape_is_refused(double, shape):
    from elfi_b200 import ops
    with pytest.raises(ValueError, match='VI must be a'):
        ops.dist_mahalanobis(np.ones((3, 5)), np.zeros(5), np.ones(shape))
    assert 'elfi_b200_dist_mahalanobis_thr_f64' not in double.CALLS


def test_d_above_the_limit_is_refused(double):
    from elfi_b200 import ops
    D = md.D_MAX + 1
    with pytest.raises(ValueError, match='MAHALANOBIS_D_MAX'):
        ops.dist_mahalanobis(np.ones((3, D)), np.zeros(D), np.eye(D))
    assert 'elfi_b200_dist_mahalanobis_thr_f64' not in double.CALLS


def test_node_in_a_model(double):
    cases.case_node_in_a_model()


def test_missing_kernel_message_names_mahalanobis():
    from elfi_b200 import model
    with pytest.raises(NotImplementedError, match="'mahalanobis' with VI="):
        model.host_distance_as_discrepancy('cosine', observed=None)
