"""Every row-stream kernel path of distance.cu and summaries.cu on the device, bit for bit against
NumPy / SciPy (rowstream_cases.py), with the kernel each case launches observed by torch.profiler
(CUPTI activity tracing) and compared with the path the restated dispatch predicts.  The last test
checks that every reachable registry path was launched at least once."""
import numpy as np
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

import rowstream_cases as cases

pytestmark = pytest.mark.gpu


def _device_config():
    """(multiprocessors, shared-memory opt-in) of cuda:0, which the table is generated for; without
    a device (collection only: every test here is skipped) the H100 SXM's."""
    if not torch.cuda.is_available():
        return cases.NOMINAL
    props = torch.cuda.get_device_properties(0)
    return props.multi_processor_count, props.shared_memory_per_block_optin


SM, OPTIN = _device_config()
CASES = cases.table(SM, OPTIN)


@pytest.fixture(scope='module', autouse=True)
def live_config():
    """(sm_count, smem_optin) the library runs with: elfi_b200_ctx_sm_count must agree with the
    count the table's wrap rows were generated for, and the restatement predicts with these."""
    from elfi_b200 import _lib
    from elfi_b200 import device as dev
    sm = int(_lib.load().elfi_b200_ctx_sm_count(dev.context()))
    assert (sm, torch.cuda.current_device()) == (SM, 0), 'the table was generated for cuda:0'
    saved = list(cases.CONFIG)
    cases.CONFIG[:] = [sm, OPTIN]
    yield sm, OPTIN
    cases.CONFIG[:] = saved


ATTEMPTS = 3


def observed(fn):
    """Run fn under CUPTI activity tracing; the set of registry paths it launched, and every
    kernel name.  Now and then the trace comes back without the library's kernel record while it
    keeps the copies and torch's own fill kernels.  When no registry kernel was recorded at all,
    fn runs again under a fresh trace (it is deterministic, and its output checks already showed
    that some kernel wrote every promised cell); a wrong kernel is a record, and fails at once."""
    for _ in range(ATTEMPTS):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        got = cases.paths_in(names)
        if got:
            break
    return got, names


def _check_path(case, fn, optin):
    want = cases.predict(case, optin)
    got, names = observed(fn)
    assert got == want, '{}: the dispatch launched {} where the restatement predicts {} ' \
        '(kernels: {})'.format(case.ident(), sorted(got), sorted(want), names)


@pytest.mark.parametrize('case', CASES, ids=[c.ident() for c in CASES])
def test_path_case(case, live_config):
    sm, optin = live_config
    if case.wrap:
        w, ns, G = cases.ring(case, optin)
        assert (-(-case.B // cases.RS_BOX_ROWS) // (sm * w)) * G > 2 * ns, \
            '{} no longer wraps the ring on this device'.format(case.ident())
    _check_path(case, lambda: cases.run(case), optin)


@pytest.mark.parametrize('n', [50, 20, 100, 300, 15])
@pytest.mark.parametrize('cols', [(1, 0, 3), (-1, 1, 2), (0, -1, 2), (2, 0, 4)])
def test_meanvar_output_columns(n, cols, live_config):
    case = cases.Case(family='meanvar', D=n, ld=n, off=0, B=67, layout='contig', wrap=False)
    _check_path(case, lambda: cases.meanvar_columns(case, *cols), live_config[1])


@pytest.mark.parametrize('route', sorted(cases.MOMENT_ROUTES))
@pytest.mark.parametrize('kind', cases.ACCURACY_KINDS)
def test_column_moments_bound(kind, route, live_config):
    optin = live_config[1]
    box = {}
    got, names = observed(lambda: box.setdefault('case', cases.moments_accuracy(kind, route)))
    want = cases.predict(box['case'], optin)
    if route == 'colmoments':
        want = {'mom:colmoments'}
    assert got == want, (sorted(got), sorted(want), names)
    if route != 'colmoments':
        assert ('/12w' if route == 'fused12' else '/8w') in ''.join(got)


def test_transposed_out_is_refused():
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    y = dev.to_device(np.random.RandomState(0).randn(9, 20))
    with pytest.raises(ValueError):
        ops.meanvar(y, out=dev.empty((2, 9)).T)
    with pytest.raises(ValueError):
        ops.autocov(y, lags=(1, 2), out=dev.empty((9, 4))[:, ::2])
    with pytest.raises(ValueError):
        ops.meanvar(y, out=torch.empty((9, 2), dtype=torch.float64))        # host memory
    with pytest.raises(ValueError):
        ops.count_zeros(y, out=dev.empty((1,)).expand(9))
    S = dev.full((9, 3), np.nan)
    ops.meanvar(y, out=S[:, :2])
    ops.count_zeros(y, out=S[:, 2])
    y_h = y.cpu().numpy()
    assert np.array_equal(S.cpu().numpy(), np.column_stack(
        [np.mean(y_h, axis=1), np.var(y_h, axis=1), np.sum(y_h == 0, axis=1)]))


def test_every_path_launched(live_config):
    """Every reachable registry path launches: one small case per path, run here, so that the check
    does not depend on which other tests of the session ran."""
    optin = live_config[1]
    rep = cases.representatives(CASES, optin)
    launched = {}
    for p in cases.reachable(optin):
        if p in rep:
            got, _ = observed(lambda: cases.run(rep[p]))
            if p in got:
                launched[p] = rep[p].ident()
        print('launched {:32s} by {}'.format(p, launched.get(p, '-')))
    missing = sorted(set(cases.reachable(optin)) - set(launched))
    assert not missing, 'never launched: {}'.format(missing)
