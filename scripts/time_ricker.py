#!/usr/bin/env python
"""CUDA-event timings of the Ricker kernels at B = 1e6 rows, n_obs = 50 (elfi_b200/csrc/ricker.cu):
the simulator with its fused summaries, the simulator alone (writing Y), the simulator followed by
ricker_summaries, for a fixed parameter (3.8, 0.3, 10) and for prior-predictive parameters (a mix
of extinct rows and high-rate rows that diverge within a warp); and ops.poisson at fixed rates.
Prints the card's name and power limit first: the numbers belong to them."""
import os
import subprocess
import sys

import numpy as np
import scipy.stats as ss
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from elfi_b200 import ops  # noqa: E402


def timeit(fn, per_batch=5, batches=7, warm=2):
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


def show(label, t):
    print('  %-44s %8.3f ms (min %.3f, max %.3f)' % (label, *t))


print('card:', card())
B, n_obs = 1_000_000, 50
rs = np.random.RandomState(0)
params = {
    'fixed (3.8, 0.3, 10)': np.tile([3.8, 0.3, 10.0], (B, 1)),
    'prior predictive': np.column_stack([np.e + rs.exponential(2.0, B),
                                         ss.truncnorm.rvs(0, 5, size=B, random_state=rs),
                                         rs.uniform(0, 100, B)]),
}
for label, P in params.items():
    P = torch.from_numpy(P).cuda()
    print('stochastic Ricker, B = 1e6, n_obs = %d, %s (data: %.0f MB)' % (n_obs, label, 8e-6 * B * n_obs))
    show('fused sim_ricker (summaries only)', timeit(lambda: ops.sim_ricker(P, n_obs, seed=1)))
    show('sim_ricker alone (writes Y)',
         timeit(lambda: ops.sim_ricker(P, n_obs, seed=1, want_data=True, want_summaries=False)))
    show('sim_ricker + ricker_summaries',
         timeit(lambda: ops.ricker_summaries(
             ops.sim_ricker(P, n_obs, seed=1, want_data=True, want_summaries=False)[0])))
    _, N, _ = ops.sim_ricker(P, n_obs, seed=1, want_latent=True, want_summaries=False)
    print('    extinct rows: %.3f, largest rate phi N: %.3g' % (
        float((N[:, -1] == 0).double().mean()), float((P[:, 2:3] * N).nan_to_num(0).max())))

r = torch.from_numpy(np.e + rs.exponential(1.0, B)).cuda()
print('deterministic Ricker, B = 1e6, n_obs = %d' % n_obs)
show('fused sim_ricker (summaries only)', timeit(lambda: ops.sim_ricker(r, n_obs, stochastic=False)))
show('sim_ricker alone (writes Y)',
     timeit(lambda: ops.sim_ricker(r, n_obs, stochastic=False, want_data=True, want_summaries=False)))

print('ops.poisson, 1e6 draws')
for lam in (0.5, 5.0, 50.0, 1e6, 1e12):
    v = torch.full((B,), lam, dtype=torch.float64, device='cuda')
    show('rate %g' % lam, timeit(lambda: ops.poisson(v, seed=1)))
