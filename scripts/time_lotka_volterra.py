#!/usr/bin/env python
"""CUDA-event timings of the Lotka-Volterra kernels (elfi_b200/csrc/lotka_volterra.cu) at the
reference's shape (50 observations over time_end = 30): the simulator and the summaries at the
true parameters (1.0, 0.005, 0.6, 50, 100) and at prior draws, B = 1e5 and 1e6, with the events
per second (the sum of n_events over the kernel time); a throughput-mode Rejection; then the rows/s
of this package's host path for comparison.  Prints the card's name and power limit first: the
numbers belong to them."""
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
from elfi_b200.examples import lotka_volterra as lv  # noqa: E402

MAX_EVENTS = 2 ** 20


def timeit(fn, per_batch=1, batches=5, warm=1):
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


def prior_params(B, seed):
    rs = np.random.RandomState(seed)
    return np.column_stack([np.exp(rs.uniform(-6, 2, (B, 3))), rs.normal(50, np.sqrt(50), B),
                            rs.normal(100, 10, B), np.zeros(B)])


print('card:', card())
for label, make in (('truth', lambda B: np.tile([1.0, 0.005, 0.6, 50, 100, 0.], (B, 1))),
                    ('prior draws', lambda B: prior_params(B, 1))):
    for B in (100_000, 1_000_000):
        P = torch.from_numpy(make(B)).cuda()
        t = timeit(lambda: ops.sim_lotka_volterra(P, 50, 30.0, seed=1, max_events=MAX_EVENTS))
        obs, n = ops.sim_lotka_volterra(P, 50, 30.0, seed=1, max_events=MAX_EVENTS)
        nh = n.cpu().numpy()
        events = float(nh.sum())
        print('%s, B = %.0e: sim_lotka_volterra %.3f ms (min %.3f, max %.3f), %.3g rows/s, '
              '%.3g events/s; events per row median %d, max %d, capped %d'
              % (label, B, *t, B / t[0] * 1e3, events / t[0] * 1e3, int(np.median(nh)),
                 int(nh.max()), int((nh == MAX_EVENTS).sum())))
        ts = timeit(lambda: ops.lv_summaries(obs), per_batch=3)
        print('%s, B = %.0e: lv_summaries %.3f ms (min %.3f, max %.3f), %.3g rows/s'
              % (label, B, *ts, B / ts[0] * 1e3))
        del P, obs, n
        torch.cuda.empty_cache()

m, _ = lv.get_device_model(seed_obs=2)
elfi.Rejection(m['d'], batch_size=100_000, seed=1).sample(100, quantile=0.01, bar=False)
torch.cuda.synchronize()
t0 = time.perf_counter()
res = elfi.Rejection(m['d'], batch_size=100_000, seed=2).sample(10_000, quantile=0.01, bar=False)
torch.cuda.synchronize()
dt = time.perf_counter() - t0
print('throughput-mode Rejection (prior draws), 1e6 simulations (10000 accepted): %.3f s, '
      '%.3g simulations/s' % (dt, res.n_sim / dt))

for label, prm, n_host in (('truth', [1.0, 0.005, 0.6, 50, 100, 0.], 100), ('prior draws', None, 100)):
    P = prior_params(n_host, 2) if prm is None else np.tile(prm, (n_host, 1))
    t0 = time.perf_counter()
    x = lv.lotka_volterra(*P.T, n_obs=50, batch_size=n_host, random_state=np.random.RandomState(0))
    dt = time.perf_counter() - t0
    print('host examples.lotka_volterra, %s, B = %d: %.3f s, %.3g rows/s' % (label, n_host, dt,
                                                                              n_host / dt))
