#!/usr/bin/env python
"""CUDA-event timings of the day care kernels (elfi_b200/csrc/daycare.cu) at the reference's shape
(29 DCCs of 53 children, 33 strains, 36 observed, time_end = 10): the fused simulator at the true
parameters (3.6, 0.6, 0.1) and at prior draws, B = 1e4 and 1e5, with the transitions per second
(the sum over rows of K n_dcc over the kernel time); the simulator writing the data followed by
daycare_summaries; the distance; a throughput-mode Rejection; then the rows/s of this package's
host path.  Prints the card's name and power limit first: the numbers belong to them."""
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
from elfi_b200.examples import daycare as dc  # noqa: E402

TRUTH = [3.6, 0.6, 0.1]


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
    return np.column_stack([rs.uniform(0, 11, B), rs.uniform(0, 2, B), rs.uniform(0, 1, B)])


print('card:', card())
for label, make in (('truth', lambda B: np.tile(TRUTH, (B, 1))),
                    ('prior draws', lambda B: prior_params(B, 1))):
    for B in (10_000, 100_000):
        P = torch.from_numpy(make(B)).cuda()
        t = timeit(lambda: ops.sim_daycare(P, seed=1), batches=3)
        S, _, K = ops.sim_daycare(P, seed=1)
        Kh = K.cpu().numpy()
        print('%s, B = %.0e: sim_daycare (fused) %.1f ms (min %.1f, max %.1f), %.3g rows/s, '
              '%.3g transitions/s; K per row median %d, max %d'
              % (label, B, *t, B / t[0] * 1e3, float(Kh.sum()) * 29 / t[0] * 1e3,
                 int(np.median(Kh)), int(Kh.max())))
        tu = timeit(lambda: ops.daycare_summaries(
            ops.sim_daycare(P, seed=1, want_data=True, want_summaries=False)[1]), batches=3)
        print('%s, B = %.0e: sim_daycare (data) + daycare_summaries %.1f ms (min %.1f, max %.1f)'
              % (label, B, *tu))
        obs = [np.asarray(v, dtype=np.float64).reshape(1, -1) for v in S[:1].cpu().numpy()
               .reshape(4, 29)]
        td = timeit(lambda: ops.daycare_distance(S, obs, 29), per_batch=5)
        print('%s, B = %.0e: daycare_distance %.3f ms (min %.3f, max %.3f), %.3g rows/s'
              % (label, B, *td, B / td[0] * 1e3))
        del P, S, K
        torch.cuda.empty_cache()

m, _ = dc.get_device_model(seed_obs=2)
elfi.Rejection(m['d'], batch_size=20_000, seed=1).sample(10, quantile=0.01, bar=False)
torch.cuda.synchronize()
t0 = time.perf_counter()
res = elfi.Rejection(m['d'], batch_size=20_000, seed=2).sample(1_000, quantile=0.01, bar=False)
torch.cuda.synchronize()
dt = time.perf_counter() - t0
print('throughput-mode Rejection (prior draws), %d simulations (1000 accepted): %.3f s, '
      '%.3g simulations/s' % (res.n_sim, dt, res.n_sim / dt))

for label, prm, n_host in (('truth', TRUTH, 1), ('prior draws', None, 1)):
    P = prior_params(n_host, 2) if prm is None else np.tile(prm, (n_host, 1))
    t0 = time.perf_counter()
    dc.daycare(*P.T, batch_size=n_host, random_state=np.random.RandomState(0))
    dt = time.perf_counter() - t0
    print('host examples.daycare, %s, B = %d: %.3f s, %.3g rows/s' % (label, n_host, dt,
                                                                       n_host / dt))
