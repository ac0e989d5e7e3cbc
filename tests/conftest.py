import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100)')
    config.addinivalue_line('markers', 'first_device_run: written after the last GPU session; '
                                       'ordered after the device-verified tests')


# GPU run order: kernel-level parity first (a failure there explains every failure above it),
# then operators inside the model graph, samplers, throughput mode, pools, BOLFI, multi-GPU.
_GPU_ORDER = ['test_distance_gpu', 'test_summaries_gpu', 'test_select_gpu', 'test_merge_gpu', 'test_smc_gpu',
              'test_kliep_gpu', 'test_gp_gpu', 'test_model_gpu', 'test_samplers_gpu',
              'test_throughput_gpu', 'test_store_gpu', 'test_bolfi_gpu', 'test_multigpu_gpu']


def _gpu_rank(item):
    name = os.path.splitext(os.path.basename(str(item.fspath)))[0]
    rank = _GPU_ORDER.index(name) if name in _GPU_ORDER else -1
    # tests of code that has not run on a device yet go last, so that `-x` cannot hide a
    # regression in verified code behind them (the marker is removed once they have passed)
    if item.get_closest_marker('first_device_run') is not None:
        rank += 100
    return rank


def pytest_collection_modifyitems(config, items):
    items.sort(key=_gpu_rank)          # stable: CPU tests keep their order and come first
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason='no CUDA device')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope='session', autouse=True)
def _built():
    """Make sure the CUDA library and the oracle are built (no-op when up to date)."""
    import __graft_entry__ as g
    g.build()


def load_golden(name):
    return dict(np.load(os.path.join(GOLDEN, name + '.npz'), allow_pickle=False))


@pytest.fixture
def golden():
    return load_golden


@pytest.fixture
def cpu_double(monkeypatch):
    """Host-logic tests without a GPU: the C ABI is replaced by tests/abi_double.py (NumPy + the
    oracle on host pointers) and device allocations by CPU tensors.  Test-only; see that module."""
    import abi_double
    abi_double.install(monkeypatch)
    return abi_double
