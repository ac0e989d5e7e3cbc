#!/usr/bin/env python
"""CUDA-event timings of the AR(1) simulator (elfi_b200/csrc/ar1.cu) at the reference's shape
(200 observations) and the true parameter phi = 0.9, at B = 1e6 and 1e7: the simulator with the
Euclidean distance to the observed series fused (one double per row written), the unfused chain
(the simulator writing the series, then dist_euclid of it) and the simulator alone; then a
throughput-mode Rejection, and the rows/s of this package's host path
(get_model(...).generate(B, outputs=['d'])) at B = 1e5.  Prints the card's name and power limit
first: the numbers belong to them."""
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
from elfi_b200.examples import ar1  # noqa: E402

N_OBS = 200


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
    print('  %-56s %9.3f ms (min %.3f, max %.3f)  %.3g rows/s' % (label, *t, B / t[0] * 1e3))


if not torch.cuda.is_available():
    sys.exit('time_ar1.py measures on a GPU; none is available')
print('card:', card())
y = torch.from_numpy(ar1.AR1(0.9, n_obs=N_OBS, random_state=np.random.RandomState(1))[0]).cuda()
for B in (1_000_000, 10_000_000):
    phi = torch.full((B,), 0.9, dtype=torch.float64, device='cuda')
    thr = 15.0
    print('AR(1), B = %.0e, %d observations' % (B, N_OBS))
    show('fused sim_ar1 (distance + acceptance, no data)',
         timeit(lambda: ops.sim_ar1(phi, N_OBS, seed=1, obs=y, thresholds=thr)), B)
    show('unfused: sim_ar1 writing X, then dist_euclid + acceptance',
         timeit(lambda: ops.dist_euclid(ops.sim_ar1(phi, N_OBS, seed=1)[0], y, thresholds=thr)), B)
    show('sim_ar1 alone (writes X)', timeit(lambda: ops.sim_ar1(phi, N_OBS, seed=1)), B)
    X = ops.sim_ar1(phi, N_OBS, seed=1)[0]
    show('dist_euclid + acceptance of X', timeit(lambda: ops.dist_euclid(X, y, thresholds=thr)), B)
    del phi, X
    torch.cuda.empty_cache()

m, _ = ar1.get_device_model(seed_obs=1)
elfi.Rejection(m['d'], batch_size=1_000_000, seed=1).sample(100, quantile=0.001, bar=False)
torch.cuda.synchronize()
t0 = time.perf_counter()
res = elfi.Rejection(m['d'], batch_size=1_000_000, seed=2).sample(10_000, quantile=0.001, bar=False)
torch.cuda.synchronize()
dt = time.perf_counter() - t0
print('throughput-mode Rejection, 1e7 simulations (10000 accepted): %.3f s, %.3g simulations/s' % (
    dt, res.n_sim / dt))

mh = ar1.get_model(seed_obs=1)
mh.generate(1000, outputs=['d'], seed=2)
B = 100_000
t0 = time.perf_counter()
d = mh.generate(B, outputs=['d'], seed=3)['d']
torch.cuda.synchronize()
dt = time.perf_counter() - t0
print('host examples.ar1 get_model().generate(%d, outputs=[\'d\']): %.3f s, %.3g rows/s' % (
    B, dt, B / dt))
