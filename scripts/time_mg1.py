#!/usr/bin/env python
"""CUDA-event timings of the M/G/1 kernels (elfi_b200/csrc/mg1.cu) at the reference's shape (50
observations, 10 quantiles) and the true parameters (1, 5, 0.2), over a range of B: the fused
simulator (quantiles only), the unfused chain (the simulator writing the data, then row_quantiles
of it) and its two halves; then a throughput-mode Rejection, the rows/s of this package's host
path (get_model(...).generate(B, outputs=['d'])), and the joint prior log density of the
hierarchical prior with sources against the same table without them.  Prints the card's name and
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
from elfi_b200.examples import mg1  # noqa: E402

Q = np.linspace(0, 1, 10)


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
    Y, _ = ops.sim_mg1(P, 50, Q, seed=1, want_data=True, want_summaries=False)
    return ops.row_quantiles(Y, Q)


print('card:', card())
for B in (100_000, 1_000_000, 10_000_000):
    P = torch.from_numpy(np.tile([1., 5., 0.2], (B, 1))).cuda()
    print('M/G/1, B = %.0e, 50 observations, 10 quantiles' % B)
    show('fused sim_mg1 (10 quantiles, no data)', timeit(lambda: ops.sim_mg1(P, 50, Q, seed=1)), B)
    show('unfused: sim_mg1 writing Y, then row_quantiles', timeit(lambda: chain(P)), B)
    show('sim_mg1 alone (writes Y)', timeit(lambda: ops.sim_mg1(
        P, 50, Q, seed=1, want_data=True, want_summaries=False)), B)
    Y, _ = ops.sim_mg1(P, 50, Q, seed=1, want_data=True, want_summaries=False)
    show('row_quantiles of Y', timeit(lambda: ops.row_quantiles(Y, Q)), B)
    del P, Y
    torch.cuda.empty_cache()

m, dp = mg1.get_device_model(seed_obs=1)
elfi.Rejection(m['d'], batch_size=1_000_000, seed=1).sample(100, quantile=0.001, bar=False)
torch.cuda.synchronize()
t0 = time.perf_counter()
res = elfi.Rejection(m['d'], batch_size=1_000_000, seed=2).sample(10_000, quantile=0.001, bar=False)
torch.cuda.synchronize()
dt = time.perf_counter() - t0
print('throughput-mode Rejection, 1e7 simulations (10000 accepted): %.3f s, %.3g simulations/s' % (
    dt, res.n_sim / dt))

B = 1_000_000
rs = np.random.RandomState(0)
t1 = rs.uniform(0, 10, B)
x = torch.from_numpy(np.column_stack([t1, t1 + rs.uniform(0, 10, B), rs.uniform(0, 0.5, B)])).cuda()
show('prior_logpdf with sources (t2 | t1), B = 1e6',
     timeit(lambda: ops.prior_logpdf(x, dp.specs, dp.sources), per_batch=20), B)
show('prior_logpdf of the same table without sources',
     timeit(lambda: ops.prior_logpdf(x, dp.specs), per_batch=20), B)

mh = mg1.get_model(seed_obs=1)
B = 100_000
t0 = time.perf_counter()
d = mh.generate(B, outputs=['d'], seed=3)['d']
torch.cuda.synchronize()
dt = time.perf_counter() - t0
print('host examples.mg1 get_model().generate(%d, outputs=[\'d\']): %.3f s, %.3g rows/s' % (
    B, dt, B / dt))
