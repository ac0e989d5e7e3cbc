"""The resident rejection step on the device (CandidateBuffer.bind_batch ->
elfi_b200_rejection_batch_f64, then CandidateBuffer.best) bit for bit against the C oracle and the
reference's merge: both distance paths across the compaction's edges, nested distances up to
K = 32, up to 7 extra sources, a buffer that runs out, thresholds that change between batches,
ties, the public Rejection sampler, the bench's shape, a side stream, and refused calls
(rejection_step_cases.py)."""
import numpy as np
import pytest
import torch

import rejection_step_cases as cases

pytestmark = pytest.mark.gpu


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


@pytest.mark.parametrize('thr_mode', ['host', 'device'])
def test_bench_shape(thr_mode):
    cases.case_bench_shape(thr_mode)


def test_side_stream_and_repeatability():
    """The largest path case on a side stream, then twice on the default stream: the same bits."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    runs = [cases.run_largest(lambda: torch.cuda.stream(side))]
    side.synchronize()
    runs += [cases.run_largest(), cases.run_largest()]
    for other in runs[1:]:
        for a, b in zip(runs[0], other):
            assert np.array_equal(a, b, equal_nan=True)
