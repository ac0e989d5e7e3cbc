#!/usr/bin/env python
"""CUDA-event timings of the Lorenz kernels (elfi_b200/csrc/lorenz.cu) at the reference's shape
(n_timestep = 160, n_obs = 40) and the true parameters (2.0, 0.1): the simulator with its fused
summaries at B = 1e5 and 1e6, and at B = 1e5 the simulator alone (writing the data) and the
simulator followed by lorenz_summaries; then the rows/s of this package's host path
(examples.lorenz.forecast_lorenz) for comparison.  Prints the card's name and power limit first:
the numbers belong to them."""
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from elfi_b200 import ops  # noqa: E402
from elfi_b200.examples import lorenz  # noqa: E402


def timeit(fn, per_batch=3, batches=7, warm=2):
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
    P = torch.from_numpy(np.tile([2.0, 0.1], (B, 1))).cuda()
    print('Lorenz, B = %.0e, n_timestep = 160, n_obs = 40 (data: %.1f GB)' % (B, 51200e-9 * B))
    show('fused sim_lorenz (summaries only)', timeit(lambda: ops.sim_lorenz(P, seed=1)), B)
    if B == 100_000:
        show('sim_lorenz alone (writes X)',
             timeit(lambda: ops.sim_lorenz(P, seed=1, want_data=True, want_summaries=False)), B)
        X = ops.sim_lorenz(P, seed=1, want_data=True, want_summaries=False)[0]
        show('lorenz_summaries of X', timeit(lambda: ops.lorenz_summaries(X)), B)
        del X
        show('sim_lorenz + lorenz_summaries',
             timeit(lambda: ops.lorenz_summaries(
                 ops.sim_lorenz(P, seed=1, want_data=True, want_summaries=False)[0])), B)
    del P
    torch.cuda.empty_cache()

n_host = 2000
t0 = time.perf_counter()
lorenz.forecast_lorenz(2.0, 0.1, batch_size=n_host, random_state=np.random.RandomState(0))
dt = time.perf_counter() - t0
print('host examples.lorenz.forecast_lorenz, %d rows: %.3f s, %.3g rows/s (NumPy)' % (
    n_host, dt, n_host / dt))
