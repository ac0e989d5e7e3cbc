#!/usr/bin/env python
"""CUDA-event timings of the scratch assay kernel (elfi_b200/csrc/scratch_assay.cu) at the
reference's shape (27 x 36 lattice, 100 cells in the first 10 rows, 288 iterations, 144
observations), at the true parameters (0.25, 0.002) and at prior draws, B = 1e4 and 1e5: the fused
simulator (summaries only), and at B = 1e4 the simulator writing the frames followed by
scratch_assay_summaries of them.  Rows/s, and kept events/s estimated from the frames' cell counts
(cells at each frame x iterations per frame x (min(pm, 1) + min(pp, 1)), on the first 1000 rows).
Then a throughput-mode Rejection and the rows/s of the host path.  Prints the card's name and
power limit first: the numbers belong to them."""
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import elfi_b200 as elfi  # noqa: E402
from elfi_b200 import ops  # noqa: E402
from elfi_b200.examples import scratch_assay as sa  # noqa: E402


def timeit(fn, per_batch=3, batches=5, warm=1):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(batches):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(per_batch):
            fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) / per_batch)
    return float(np.median(ts)), float(min(ts)), float(max(ts))


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                            '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        return q.stdout.strip() or torch.cuda.get_device_name(0)
    except OSError:
        return torch.cuda.get_device_name(0) + ' (power limit not read)'


def kept_events_per_row(P, init):
    """Estimated kept motility and proliferation slots per row, from the frames of the first
    1000 rows."""
    P = P[:1000]
    X, _ = ops.sim_scratch_assay(P, init, seed=1, want_data=True, want_summaries=False)
    counts = X.sum(dim=(1, 2)).double()[:, :-1]             # cells at the start of each frame
    p = P.clamp(0, 1).sum(dim=1)
    return float((counts.sum(dim=1) * 2 * p).mean())


def show(label, t, B, events=None):
    extra = '' if events is None else ', %.3g kept events/s' % (events * B / t[0] * 1e3)
    print('  %-52s %9.3f ms (min %.3f, max %.3f)  %.3g rows/s%s' % (label, *t, B / t[0] * 1e3,
                                                                     extra))


def chain(P, init):
    X, _ = ops.sim_scratch_assay(P, init, seed=1, want_data=True, want_summaries=False)
    return ops.scratch_assay_summaries(X)


print('card:', card())
obs, init, _ = sa._observed(None, None, None, 1)
rs = np.random.RandomState(0)
for B in (10_000, 100_000):
    prior = rs.uniform(0, 1, (B, 2))
    for label, P in (('truth', np.tile((0.25, 0.002), (B, 1))), ('prior draws', prior)):
        P = torch.from_numpy(P).cuda()
        ev = kept_events_per_row(P, init)
        print('scratch assay at the %s, B = %.0e (about %.0f kept events per row)' % (label, B, ev))
        show('fused sim_scratch_assay (summaries; no frames)',
             timeit(lambda: ops.sim_scratch_assay(P, init, seed=1)), B, ev)
        if B == 10_000:
            show('unfused: frames, then scratch_assay_summaries', timeit(lambda: chain(P, init)), B,
                 ev)
        del P
    torch.cuda.empty_cache()

m, dp = sa.get_device_model(seed_obs=1)
elfi.Rejection(m['d'], batch_size=100_000, seed=1).sample(10, quantile=0.001, bar=False)
torch.cuda.synchronize()
t0 = time.perf_counter()
res = elfi.Rejection(m['d'], batch_size=100_000, seed=2).sample(300, quantile=0.001, bar=False)
torch.cuda.synchronize()
dt = time.perf_counter() - t0
print('throughput-mode Rejection, %d simulations (300 accepted): %.3f s, %.3g simulations/s' % (
    res.n_sim, dt, res.n_sim / dt))

mh = sa.get_model(seed_obs=1)
B = 20
t0 = time.perf_counter()
mh.generate(B, outputs=['d'], seed=3)
dt = time.perf_counter() - t0
print('host examples.scratch_assay get_model().generate(%d, outputs=[\'d\']): %.3f s, %.3g rows/s'
      % (B, dt, B / dt))
