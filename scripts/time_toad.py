#!/usr/bin/env python
"""CUDA-event timings of the toad kernels (elfi_b200/csrc/toad.cu) at the reference's shape
(66 toads, 63 days) and the true parameters (1.7, 35, 0.6): at B = 1e5 the simulator alone (writing
the data), the four lags' toad_summaries of that data, and the fused kernel; the fused kernel at
B = 1e6; a throughput-mode Rejection; then the rows/s of this package's host path for comparison.
Prints the card's name and power limit first: the numbers belong to them."""
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
from elfi_b200.examples import toad  # noqa: E402


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
    print('  %-46s %9.3f ms (min %.3f, max %.3f)  %.3g rows/s' % (label, *t, B / t[0] * 1e3))


print('card:', card())
for B in (100_000, 1_000_000):
    P = torch.from_numpy(np.tile([1.7, 35.0, 0.6], (B, 1))).cuda()
    print('toad, B = %.0e, 66 toads x 63 days (data: %.1f GB)' % (B, 33264e-9 * B))
    show('fused sim_toad (4 lags of summaries)', timeit(lambda: ops.sim_toad(P, seed=1)), B)
    if B == 100_000:
        show('sim_toad alone (writes X)',
             timeit(lambda: ops.sim_toad(P, seed=1, want_data=True, lags=None)), B)
        X = ops.sim_toad(P, seed=1, want_data=True, lags=None)[0].permute(1, 2, 0)
        show('toad_summaries of X, 4 lags',
             timeit(lambda: [ops.toad_summaries(X, lag) for lag in (1, 2, 4, 8)]), B)
        for lag in (1, 8):
            show('toad_summaries of X, lag %d' % lag, timeit(lambda: ops.toad_summaries(X, lag)), B)
        Z = torch.zeros_like(X)
        show('toad_summaries, every toad returned (lag 1)',
             timeit(lambda: ops.toad_summaries(Z, 1)), B)
        del X, Z
    del P
    torch.cuda.empty_cache()

m, _ = toad.get_device_model(seed_obs=2)
rej = elfi.Rejection(m['d'], batch_size=100_000, seed=1)
rej.sample(100, quantile=0.01, bar=False)
torch.cuda.synchronize()
t0 = time.perf_counter()
res = elfi.Rejection(m['d'], batch_size=100_000, seed=2).sample(10_000, quantile=0.01, bar=False)
torch.cuda.synchronize()
dt = time.perf_counter() - t0
print('throughput-mode Rejection, 1e6 simulations (10000 accepted): %.3f s, %.3g simulations/s' % (
    dt, res.n_sim / dt))

n_host = 500
t0 = time.perf_counter()
x = toad.toad(1.7, 35.0, 0.6, batch_size=n_host, random_state=np.random.RandomState(0))
t1 = time.perf_counter()
for lag in (1, 2, 4, 8):
    toad.compute_summaries(x, lag)
t2 = time.perf_counter()
print('host examples.toad, %d rows: simulate %.3f s, summaries %.3f s, %.3g rows/s end to end' % (
    n_host, t1 - t0, t2 - t1, n_host / (t2 - t0)))
