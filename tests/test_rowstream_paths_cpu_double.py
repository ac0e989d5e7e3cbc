"""The row-stream case bodies of rowstream_cases.py against the CPU test double (NumPy and the
oracle behind the C ABI): the checkers accept correct results at every layout, row count and output
configuration.  Which kernel would run is the device tests' business; the wrap row counts only
exercise the device's ring and are left to them."""
import numpy as np
import pytest
import torch

import rowstream_cases as cases

pytestmark = pytest.mark.usefixtures('cpu_double')

CASES = [c for c in cases.table(*cases.NOMINAL) if not c.wrap]


@pytest.fixture(autouse=True)
def doubles(cpu_double, monkeypatch):
    """The segmented distances of testbench_double.py on top of the C ABI double, and the moments
    bound at the depth of the order the double restates: colmoments_f64's, for every route (the
    fused kernel's own order is checked on the device)."""
    import abi_double
    import testbench_double
    abi_double.install(monkeypatch, testbench_double.TABLE)
    monkeypatch.setattr(cases, 'moments_depth', lambda case, B, sm=None, optin=None:
                        cases.colmoments_depth(case.D, B, cpu_double.SM_COUNT))


@pytest.mark.parametrize('case', CASES, ids=[c.ident() for c in CASES])
def test_path_case(case):
    cases.run(case)


@pytest.mark.parametrize('n', [50, 20, 100, 300, 15])
@pytest.mark.parametrize('cols', [(1, 0, 3), (-1, 1, 2), (0, -1, 2), (2, 0, 4)])
def test_meanvar_output_columns(n, cols):
    case = cases.Case(family='meanvar', D=n, ld=n, off=0, B=67, layout='contig', wrap=False)
    cases.meanvar_columns(case, *cols)


@pytest.mark.parametrize('route', sorted(cases.MOMENT_ROUTES))
@pytest.mark.parametrize('kind', cases.ACCURACY_KINDS)
def test_column_moments_bound(kind, route):
    cases.moments_accuracy(kind, route)


def test_transposed_out_is_refused():
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    y = dev.to_device(np.random.RandomState(0).randn(9, 20))
    with pytest.raises(ValueError):
        ops.meanvar(y, out=dev.empty((2, 9)).T)
    with pytest.raises(ValueError):
        ops.autocov(y, lags=(1, 2), out=dev.empty((2, 9)).T)
    with pytest.raises(ValueError):
        ops.autocov(y, lags=(1, 2), out=dev.empty((9, 4))[:, ::2])
    with pytest.raises(ValueError):
        ops.meanvar(y, out=dev.empty((8, 2)))
    with pytest.raises(ValueError):
        ops.meanvar(y, out=dev.empty((9, 2), dtype=torch.float32))
    with pytest.raises(ValueError):
        ops.count_zeros(y, out=dev.empty((9, 1)))
    with pytest.raises(ValueError):
        ops.count_zeros(y, out=dev.empty((1,)).expand(9))
    S = dev.empty((9, 3))
    ops.meanvar(y, out=S[:, :2])          # a column slice of a wider matrix is fine
