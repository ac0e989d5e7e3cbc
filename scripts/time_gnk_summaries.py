#!/usr/bin/env python
"""CUDA-event timings of the g-and-k robust summaries at B = 1e6 rows (elfi_b200/csrc/gnkstats.cu):
the fused simulator + summaries against the unfused chain (simulator, then gnk_summaries) and
against the simulator + rowsort of the order-statistic path.  Univariate n_obs 50 and 256,
bivariate n_obs 150.  Prints the card's name and power limit first: the numbers belong to them."""
import os
import subprocess
import sys

import numpy as np
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
B = 1_000_000
rs = np.random.RandomState(0)
cols = [torch.from_numpy(v).cuda() for v in (rs.uniform(0, 10, B), rs.uniform(0.1, 10, B),
                                             rs.uniform(0, 10, B), rs.uniform(0, 10, B))]
for n_obs in (50, 256):
    print('univariate g-and-k, B = 1e6, n_obs = %d (data: %.0f MB)' % (n_obs, 8e-6 * B * n_obs))
    show('fused sim_gnk_summaries (ss_robust)',
         timeit(lambda: ops.sim_gnk_summaries(*cols, n_obs=n_obs, seed=1, kind='ss_robust')))
    show('sim_gnk + gnk_summaries (ss_robust)',
         timeit(lambda: ops.gnk_summaries(ops.sim_gnk(*cols, n_obs=n_obs, seed=1), 'ss_robust')))
    show('sim_gnk + rowsort', timeit(lambda: ops.rowsort(ops.sim_gnk(*cols, n_obs=n_obs, seed=1))))
    show('sim_gnk alone', timeit(lambda: ops.sim_gnk(*cols, n_obs=n_obs, seed=1)))

P = torch.from_numpy(np.column_stack(
    [rs.uniform(0, 5, B), rs.uniform(0, 5, B), rs.uniform(0.01, 5, B), rs.uniform(0.01, 5, B),
     rs.uniform(-5, 5, B), rs.uniform(-5, 5, B), rs.uniform(-.5, 5, B), rs.uniform(-.5, 5, B),
     rs.uniform(-1, 1, B)])).cuda()
n_obs = 150
print('bivariate g-and-k, B = 1e6, n_obs = %d (data: %.0f MB)' % (n_obs, 16e-6 * B * n_obs))
show('fused sim_bignk (ss_robust)',
     timeit(lambda: ops.sim_bignk(P, n_obs=n_obs, seed=1, want_data=False, kind='ss_robust')))
show('sim_bignk + gnk_summaries (ss_robust)',
     timeit(lambda: ops.gnk_summaries(ops.sim_bignk(P, n_obs=n_obs, seed=1)[0], 'ss_robust')))
show('sim_bignk + transposed copy + rowsort',
     timeit(lambda: ops.rowsort(ops.sim_bignk(P, n_obs=n_obs, seed=1)[0].permute(0, 2, 1)
                                .reshape(2 * B, n_obs))))
show('sim_bignk alone', timeit(lambda: ops.sim_bignk(P, n_obs=n_obs, seed=1)))
