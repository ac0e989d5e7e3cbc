"""Plugin boundaries of SURVEY.md section 8b, checked against the golden results of the
UNMODIFIED reference (tests/golden/, generated with the reference's own samplers and seeds):
  * #2 the client: elfi_b200.client.Client driven in the reference's BatchHandler protocol
    (CPU, ABI test double);
  * #1 the operators: a model whose Distance and Summary operations are the ctypes stubs of
    integration/elfi_b200_ops.py (INTEGRATION.md section B) under host-RNG Rejection and SMC --
    GPU test, against the goldens; the stubs alone against SciPy / NumPy."""
import os
import sys
from functools import partial

import numpy as np
import pytest

from conftest import load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _stub_model():
    """Config #1's MA2 model with the ctypes stubs of integration/elfi_b200_ops.py as its Summary
    and Distance operations -- the nodes a maintainer of the reference would declare
    (INTEGRATION.md section B).  The distance stub gets the summaries as the host matrix that the
    reference's np.column_stack hands to cdist (elfi/model/utils.py:37-52)."""
    from elfi_b200 import device as dev
    from elfi_b200 import model as em
    from elfi_b200.examples import ma2
    sys.path.insert(0, os.path.join(ROOT, 'integration'))
    import elfi_b200_ops as b200
    y = ma2.MA2(.6, .2, random_state=np.random.RandomState(4))
    m = em.ElfiModel()
    em.Prior(ma2.CustomPrior1, 2, model=m, name='t1')
    em.Prior(ma2.CustomPrior2, m['t1'], 1, name='t2')
    em.Simulator(partial(ma2.MA2, n_obs=100), m['t1'], m['t2'], observed=y, name='MA2')
    em.Summary(b200.device_autocov, m['MA2'], name='S1')
    em.Summary(partial(b200.device_autocov, lag=2), m['MA2'], name='S2')
    em.Distance(lambda XA, XB: b200.device_cdist_euclidean(dev.to_host(XA), XB), m['S1'], m['S2'],
                name='d')
    return m


@pytest.mark.gpu
def test_reference_rejection_with_device_operators():
    """Rejection and SMC (host RNG, the reference's seeds) on a model whose Summary / Distance
    operations are the device stubs: the reference's golden results (tests/golden/gen_golden.py)."""
    import elfi_b200 as elfi
    from test_samplers_gpu import _check_smc
    m = _stub_model()
    g = load_golden('ma2_rejection_quantile')
    res = elfi.Rejection(m['d'], batch_size=1000, seed=123).sample(100, quantile=0.01, bar=False)
    assert res.n_sim == int(g['n_sim']) and res.threshold == float(g['threshold'])
    assert np.array_equal(res.discrepancies, g['out_d'])
    assert np.array_equal(res.samples['t1'], g['out_t1'])
    assert np.array_equal(res.samples['t2'], g['out_t2'])
    # SMC on the same model: the first population bit for bit, the later ones at the parity bar of
    # the device SMC (its importance weights come from the mixture-density kernel)
    gs = load_golden('ma2_smc_thresholds')
    smc = elfi.SMC(m['d'], batch_size=1000, seed=20).sample(150, thresholds=[.6, .3, .15],
                                                            bar=False)
    _check_smc(smc, gs)


@pytest.mark.gpu
def test_device_operator_stubs_match_scipy():
    """The ctypes stubs of integration/elfi_b200_ops.py alone, against SciPy / NumPy."""
    sys.path.insert(0, os.path.join(ROOT, 'integration'))
    import elfi_b200_ops as b200
    from scipy.spatial.distance import cdist
    rs = np.random.RandomState(5)
    S, obs, w = rs.randn(3000, 128), rs.randn(1, 128), rs.rand(128)
    assert np.array_equal(b200.device_cdist_euclidean(S, obs), cdist(S, obs, 'euclidean'))
    assert np.array_equal(b200.device_cdist_euclidean(S, obs, w=w), cdist(S, obs, 'euclidean', w=w))
    x = rs.randn(500, 100)
    assert np.array_equal(b200.device_autocov(x, 2), np.mean(x[:, 2:] * x[:, :-2], axis=1))


def test_client_runs_reference_rejection(cpu_double):
    """The client as the reference's BatchHandler drives it (elfi/client.py:150-182): one task per
    batch submitted in index order, `num_cores` batches in flight, results claimed by task id in
    submission order.  The MA2 batches of config #1 (elfi_b200's model on the ABI test double)
    merged into the best 100 give the reference's golden Rejection result."""
    from elfi_b200 import model as em
    from elfi_b200.client import Client
    from elfi_b200.examples import ma2
    g = load_golden('ma2_rejection_quantile')
    client = Client(devices=[0])
    assert client.num_cores == 1
    m = ma2.get_model(seed_obs=4)
    context = em.ComputationContext(batch_size=1000, seed=123)
    plan = em.compile_plan(m, ['d'])
    n_batches = int(g['n_sim']) // context.batch_size
    pending, d = [], []
    for b in range(n_batches + 1):
        if b < n_batches:
            pending.append(client.apply(em.execute_batch, m, ['d'], context, b, compiled=plan))
        if len(pending) > client.num_cores or (b == n_batches and pending):
            batch = client.get_result(pending.pop(0))
            d.append(np.asarray(batch['d'].cpu()).ravel())
    assert not pending and not client.tasks and len(d) == n_batches
    d = np.concatenate(d)
    best = np.sort(d)[:len(g['out_d'])]
    assert len(d) == int(g['n_sim'])
    assert np.array_equal(best, np.ravel(g['out_d'])) and best[-1] == float(g['threshold'])


def test_client_task_api():
    from elfi_b200.client import Client
    c = Client(devices=[0])
    a = c.apply(lambda x, y=1: x + y, 2, y=3)
    b = c.apply(lambda: 7)
    assert c.is_ready(a) and c.num_cores == 1
    c.remove_task(b)
    assert c.get_result(a) == 5
    with pytest.raises(KeyError):
        c.get_result(b)
    assert c.apply_sync(lambda: 'ok') == 'ok'
    c.reset()
    assert not c.tasks


@pytest.mark.gpu
def test_client_spreads_batches_over_devices():
    """Two worker threads (both on GPU 0 here, any two GPUs on a bigger box): tasks land on
    devices round-robin, run concurrently and come back by id."""
    import threading
    import torch
    from elfi_b200.client import Client
    n = min(2, torch.cuda.device_count())
    c = Client(devices=list(range(n)) if n == 2 else [0, 0])
    assert c.num_cores == 2
    seen = []

    def task(i):
        seen.append((i, torch.cuda.current_device(), threading.get_ident()))
        return torch.full((4,), float(i), device='cuda').sum().item()
    ids = [c.apply(task, i) for i in range(6)]
    assert [c.get_result(t) for t in ids] == [4.0 * i for i in range(6)]
    assert len({ident for _, _, ident in seen}) == 2
    for i, device, _ in seen:
        assert device == c.devices[i % 2]
