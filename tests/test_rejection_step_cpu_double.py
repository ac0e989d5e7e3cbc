"""The resident rejection step's case bodies (rejection_step_cases.py) against the CPU test double
(NumPy and the oracle behind the C ABI): the checkers accept a correct step at every shape,
source layout, capacity and threshold they pose.  The bench-scale case and the stream case are the
device tests' business."""
import pytest

import rejection_step_cases as cases

pytestmark = pytest.mark.usefixtures('cpu_double')


@pytest.mark.parametrize('path,D,ld,B', cases.SHAPES)
def test_path_and_shape(path, D, ld, B):
    cases.case_path_shape(path, D, ld, B)


@pytest.mark.parametrize('path', ['rowstream', 'direct'])
@pytest.mark.parametrize('K', cases.NESTED_K)
def test_nested(K, path):
    cases.case_nested(K, path)


def test_default_key_is_reference_key():
    cases.case_default_key_is_reference_key()


@pytest.mark.parametrize('n_extra', cases.N_EXTRA)
def test_extras(n_extra):
    cases.case_extras(n_extra)


@pytest.mark.parametrize('kind', cases.CAPACITY_KINDS)
def test_capacity(kind):
    cases.case_capacity(kind)


@pytest.mark.parametrize('kind', cases.THRESHOLD_KINDS)
def test_thresholds(kind):
    cases.case_thresholds(kind)


def test_best_ties():
    cases.case_best_ties()


@pytest.mark.parametrize('kind', cases.RAW_KINDS)
def test_raw_append(kind):
    cases.case_raw_append(kind)


def test_public_rejection():
    cases.case_public_rejection()


def test_refusals():
    cases.case_refusals()
