"""The SMC accuracy cases of smc_cases.py against the CPU test double (NumPy and the oracle behind
the C ABI): the references, bounds and shape plumbing hold for a correct implementation.  The
shapes with 1e6 points or components are left to the device."""
import pytest

import smc_cases as cases

pytestmark = pytest.mark.usefixtures('cpu_double')

CPU_M = [m for m in cases.CHUNK_M if m < 100_000]
CPU_WS_N = [n for n in cases.WS_N if n < 1_000_000]


@pytest.mark.parametrize('p', cases.TEMPLATED_P)
def test_gm_templated_kernel(p):
    cases.case_templated(p)


@pytest.mark.parametrize('p', [5, 8])
def test_gm_generic_kernel(p):
    cases.case_generic(p)


def test_gm_rejects_p17_and_context_survives():
    cases.case_p17_rejected()


@pytest.mark.parametrize('M', CPU_M)
def test_gm_component_chunks(M):
    cases.case_chunking(M)


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


@pytest.mark.parametrize('N', CPU_WS_N)
@pytest.mark.parametrize('p', cases.WS_P)
def test_weighted_stats_shapes(p, N):
    cases.case_weighted_stats(p, N)


@pytest.mark.parametrize('N', [1, 2, 257, 4 * 132 * 256 + 1])
@pytest.mark.parametrize('kind', cases.W_KINDS)
def test_weighted_stats_weights(kind, N):
    cases.case_weighted_stats(3, N, kind)


def test_weighted_stats_offset():
    cases.case_weighted_stats_offset(N=4097)


def test_weighted_stats_strided():
    cases.case_weighted_stats_strided()


def test_smc_weights_ulp():
    cases.case_smc_weights()
