"""The SMC population kernels of smc.cu against plain high-precision references at the accuracy
include/elfi_b200.h promises: the mixture density on both paths (fp64 and mixed) at every kernel
path, chunk and block tail, covariance and weight family, with an outlying centre, strided inputs
and near underflow, its invariance under slicing (the sharded multi-GPU density), permutation and
repetition; the weighted statistics against a derived rounding bound; the importance weights
within 2 ulp.  Shapes, references and bounds: smc_cases.py."""
import pytest

import smc_cases as cases

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    print('\nlargest relative error of q per mode: {}  (bounds: fp64 {:.3g}, mixed {:.3g})'.format(
        {k: '{:.3g}'.format(v) for k, v in cases.MEASURED.items()}, cases.FP64_BOUND,
        cases.MIXED_BOUND))


@pytest.mark.parametrize('p', cases.TEMPLATED_P)
def test_gm_templated_kernel(p):
    cases.case_templated(p)


@pytest.mark.parametrize('p', cases.GENERIC_P)
def test_gm_generic_kernel(p):
    cases.case_generic(p)


def test_gm_rejects_p17_and_context_survives():
    cases.case_p17_rejected()


@pytest.mark.parametrize('M', cases.CHUNK_M)
def test_gm_component_chunks(M):
    cases.case_chunking(M)


def test_gm_production_shape_and_shards():
    cases.case_production()


@pytest.mark.parametrize('N', cases.TAIL_N)
def test_gm_point_tails(N):
    cases.case_point_tails(N)


@pytest.mark.parametrize('p', [2, 6])
@pytest.mark.parametrize('kind', cases.COV_KINDS)
def test_gm_covariances(kind, p):
    cases.case_covariance(kind, p)


@pytest.mark.parametrize('kind', cases.W_KINDS)
def test_gm_weights(kind):
    cases.case_weights(kind)


@pytest.mark.parametrize('sd', cases.CENTRING_SD)
def test_gm_outlying_centre(sd):
    cases.case_centring(sd)


@pytest.mark.parametrize('p', [2, 5])
def test_gm_strided_inputs(p):
    cases.case_strided(p)


@pytest.mark.parametrize('p,cov', [(1, 'scalar'), (2, 'diag'), (4, 'full'), (7, 'var1e4')])
def test_gm_underflow_contract(p, cov):
    cases.case_underflow(p, cov)


@pytest.mark.parametrize('p', [1, 3, 6])
def test_gm_invariance(p):
    cases.case_invariance(p)


@pytest.mark.parametrize('N', cases.WS_N)
@pytest.mark.parametrize('p', cases.WS_P)
def test_weighted_stats_shapes(p, N):
    cases.case_weighted_stats(p, N)


@pytest.mark.parametrize('N', [1, 2, 257, 4 * 132 * 256 + 1])
@pytest.mark.parametrize('kind', cases.W_KINDS)
def test_weighted_stats_weights(kind, N):
    cases.case_weighted_stats(3, N, kind)


def test_weighted_stats_offset():
    cases.case_weighted_stats_offset()


def test_weighted_stats_strided():
    cases.case_weighted_stats_strided()


def test_smc_weights_ulp():
    cases.case_smc_weights()
