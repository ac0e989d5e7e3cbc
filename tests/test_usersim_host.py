"""User-written CUDA simulators (ops.usersim_*, tools.cuda_simulator, tools.fused_summary) without
a GPU: the limits come from elfi_b200.h, every shape is refused before NVRTC would run, and the
summary helpers read the columns they are given."""
import numpy as np
import pytest
import torch

from elfi_b200 import _lib, ops, tools
from elfi_b200.throughput import LazySimulation

SOURCE = '__device__ void simulate(const double* t, elfi::RowStream& r, double* y) { y[0] = t[0]; }'


@pytest.fixture
def no_native(monkeypatch):
    """Every call into the library fails the test: the checks must come first."""
    def call(name, *args):
        raise AssertionError('{} was called'.format(name))
    monkeypatch.setattr(_lib, 'call', call)


def test_limits_come_from_the_header():
    assert ops.USERSIM_P_MAX == _lib.CONSTANTS['USERSIM_P_MAX'] == 16
    assert ops.USERSIM_P_MAX == _lib.CONSTANTS['MAX_PRIOR_PARAMS']
    assert ops.USERSIM_N_OUT_MAX == _lib.CONSTANTS['USERSIM_N_OUT_MAX']
    assert ops.USERSIM_N_SUM_MAX == _lib.CONSTANTS['USERSIM_N_SUM_MAX']
    assert 1 <= ops.USERSIM_LOCAL_MAX <= ops.USERSIM_N_OUT_MAX


BAD_SHAPES = [
    dict(n_params=0, n_out=10), dict(n_params=17, n_out=10),
    dict(n_params=2, n_out=0), dict(n_params=2, n_out=ops.USERSIM_N_OUT_MAX + 1),
    dict(n_params=2, n_out=10, n_summaries=-1),
    dict(n_params=2, n_out=10, n_summaries=ops.USERSIM_N_SUM_MAX + 1),
    dict(n_params=2, n_out=10, salt=-1), dict(n_params=2, n_out=10, salt=2 ** 32),
    dict(n_params=2.5, n_out=10), dict(n_params=True, n_out=10), dict(n_params=2, n_out=10.5),
]


@pytest.mark.parametrize('shape', BAD_SHAPES, ids=lambda s: '-'.join(
    '{}={}'.format(k, v) for k, v in s.items()))
def test_shapes_refused_before_compiling(no_native, shape):
    with pytest.raises(ValueError, match='a user simulator takes an integer'):
        ops.usersim_compile(SOURCE, **shape)
    with pytest.raises(ValueError, match='a user simulator takes an integer'):
        tools.cuda_simulator(SOURCE, **shape)


def test_limits_are_inclusive():
    assert ops.usersim_shapes(16, ops.USERSIM_N_OUT_MAX, ops.USERSIM_N_SUM_MAX, 2 ** 32 - 1) == (
        16, ops.USERSIM_N_OUT_MAX, ops.USERSIM_N_SUM_MAX, 2 ** 32 - 1)
    assert ops.usersim_shapes(np.int64(1), 1.0) == (1, 1, 0, 0)


@pytest.mark.parametrize('source', ['', '   \n', None, b'__device__ void simulate();'])
def test_source_must_be_text(no_native, source):
    with pytest.raises(ValueError, match='non-empty string'):
        ops.usersim_compile(source, 1, 1)
    with pytest.raises(ValueError, match='non-empty string'):
        tools.cuda_simulator(source, 1, 1)


def test_simulator_checks_its_arguments_first(no_native):
    sim = tools.cuda_simulator(SOURCE, 2, 5)
    with pytest.raises(ValueError, match='takes 2 parameters, got 1'):
        sim(np.zeros(3), batch_size=3)


def test_run_refuses_what_the_simulator_cannot_give(no_native):
    sim = ops.UserSimulator(None, 0, 2, 5, 0, 0)
    with pytest.raises(ValueError, match='neither'):
        ops.usersim_run(sim, [np.zeros(3)] * 2, want_data=False, want_summaries=False)
    with pytest.raises(ValueError, match='no summaries'):
        ops.usersim_run(sim, [np.zeros(3)] * 2)
    with pytest.raises(ValueError, match='no summaries'):
        ops.usersim_summarise(sim, np.zeros(5))


def _lazy(S):
    return LazySimulation((S.shape[0], 7), lambda kind: S, lambda: None)


def test_fused_summary_reads_columns():
    S = torch.arange(12, dtype=torch.float64).reshape(4, 3)
    assert torch.equal(tools.fused_summary(1)(_lazy(S)), S[:, 1])
    assert torch.equal(tools.fused_summary([2, 0])(_lazy(S)), S[:, [2, 0]])
    assert tools.fused_summary(np.int64(0))(_lazy(S)).shape == (4,)


def test_fused_summary_of_other_data():
    with pytest.raises(ValueError, match='give it the simulator'):
        tools.fused_summary(0)(np.zeros((1, 7)))

    class Sim:
        @staticmethod
        def summarise(y):
            y = np.atleast_2d(y)
            return np.column_stack([y.sum(axis=1), y.max(axis=1)])

    y = np.arange(7.0)
    assert np.array_equal(tools.fused_summary(1, Sim)(y), [6.0])
    assert np.array_equal(tools.fused_summary([0, 1], Sim)(y), [[21.0, 6.0]])
