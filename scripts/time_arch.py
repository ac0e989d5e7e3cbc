#!/usr/bin/env python
"""CUDA-event timings of the ARCH(1) kernels (elfi_b200/csrc/arch.cu) at the reference's shape
(100 observations, 5 lags, 17 summaries) and the true parameters (0.3, 0.7), over a range of B:
the fused simulator (summaries only), the unfused chain (the simulator writing the data, then
arch_summaries of it) and the simulator alone; then a throughput-mode Rejection, and the rows/s of
this package's host path (get_model(...).generate(B, outputs=['d'])) for comparison.  Prints the
card's name and power limit first: the numbers belong to them."""
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
from elfi_b200.examples import arch  # noqa: E402


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


def show(label, t, B):
    print('  %-52s %9.3f ms (min %.3f, max %.3f)  %.3g rows/s' % (label, *t, B / t[0] * 1e3))


def chain(P):
    Y, _ = ops.sim_arch(P, 100, 5, seed=1, want_data=True, want_summaries=False)
    return ops.arch_summaries(Y, 5)


print('card:', card())
for B in (10_000, 100_000, 1_000_000, 10_000_000):
    P = torch.from_numpy(np.tile([0.3, 0.7], (B, 1))).cuda()
    print('ARCH(1), B = %.0e, 100 observations, 5 lags' % B)
    show('fused sim_arch (17 summaries, no data)', timeit(lambda: ops.sim_arch(P, seed=1)), B)
    show('unfused: sim_arch writing Y, then arch_summaries', timeit(lambda: chain(P)), B)
    show('sim_arch alone (writes Y)', timeit(lambda: ops.sim_arch(
        P, seed=1, want_data=True, want_summaries=False)), B)
    Y, _ = ops.sim_arch(P, seed=1, want_data=True, want_summaries=False)
    show('arch_summaries of Y', timeit(lambda: ops.arch_summaries(Y, 5)), B)
    del P, Y
    torch.cuda.empty_cache()

m, _ = arch.get_device_model(seed_obs=1)
elfi.Rejection(m['d'], batch_size=1_000_000, seed=1).sample(100, quantile=0.001, bar=False)
torch.cuda.synchronize()
t0 = time.perf_counter()
res = elfi.Rejection(m['d'], batch_size=1_000_000, seed=2).sample(10_000, quantile=0.001, bar=False)
torch.cuda.synchronize()
dt = time.perf_counter() - t0
print('throughput-mode Rejection, 1e7 simulations (10000 accepted): %.3f s, %.3g simulations/s' % (
    dt, res.n_sim / dt))

mh = arch.get_model(seed_obs=1)
for B in (10_000, 100_000):
    t0 = time.perf_counter()
    d = mh.generate(B, outputs=['d'], seed=3)['d']
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    print('host examples.arch get_model().generate(%d, outputs=[\'d\']): %.3f s, %.3g rows/s' % (
        B, dt, B / dt))
