#!/usr/bin/env python
"""CUDA-event timings of the stochastic volatility kernel (elfi_b200/csrc/svm.cu) at the reference's
shape (50 observations) and constants, at the true parameters (1.2, 0.5) and at prior draws, over
B = 1e4 .. 1e6: the fused simulator (kurt and skew only), the unfused chain (the simulator writing
the data, then svm_summaries of it); then a throughput-mode Rejection and the rows/s of the host
path (get_model(...).generate(B, outputs=['d'])).  Prints the card's name and power limit first:
the numbers belong to them."""
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
from elfi_b200.examples import stochastic_volatility_model as svm  # noqa: E402

FIXED = (1.0, 0.0, 0.0, 0.95, 0.2)


def timeit(fn, per_batch=5, batches=5, warm=2):
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
    Y, _ = ops.sim_svm(P, 50, seed=1, want_data=True, want_summaries=False)
    return ops.svm_summaries(Y)


print('card:', card())
rs = np.random.RandomState(0)
for B in (10_000, 100_000, 1_000_000):
    prior = np.column_stack([rs.uniform(0.5, 2.0, B), rs.uniform(-1, 1, B), np.tile(FIXED, (B, 1))])
    for label, P in (('truth', np.tile((1.2, 0.5) + FIXED, (B, 1))), ('prior draws', prior)):
        P = torch.from_numpy(P).cuda()
        print('SVM at the %s, B = %.0e, 50 observations' % (label, B))
        show('fused sim_svm (kurt, skew; no data)', timeit(lambda: ops.sim_svm(P, 50, seed=1)), B)
        show('unfused: sim_svm writing Y, then svm_summaries', timeit(lambda: chain(P)), B)
        del P
    torch.cuda.empty_cache()

m, dp = svm.get_device_model(seed_obs=1)
elfi.Rejection(m['d'], batch_size=1_000_000, seed=1).sample(100, quantile=0.001, bar=False)
torch.cuda.synchronize()
t0 = time.perf_counter()
res = elfi.Rejection(m['d'], batch_size=1_000_000, seed=2).sample(10_000, quantile=0.001, bar=False)
torch.cuda.synchronize()
dt = time.perf_counter() - t0
print('throughput-mode Rejection, 1e7 simulations (10000 accepted): %.3f s, %.3g simulations/s' % (
    dt, res.n_sim / dt))

mh = svm.get_model(seed_obs=1)
B = 10_000
t0 = time.perf_counter()
d = mh.generate(B, outputs=['d'], seed=3)['d']
dt = time.perf_counter() - t0
print('host examples.stochastic_volatility_model get_model().generate(%d, outputs=[\'d\']): '
      '%.3f s, %.3g rows/s' % (B, dt, B / dt))
