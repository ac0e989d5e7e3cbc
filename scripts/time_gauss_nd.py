#!/usr/bin/env python
"""CUDA-event timings of the n-D Gaussian mean simulator (elfi_b200/csrc/gauss_nd.cu) at B = 1e6,
D in {1, 2, 4, 8, 16} and n_obs in {15, 50}: the simulator with its [means | variances] fused (no
data written), and the data materialised by the simulator followed by the summary kernel.  Each
line carries the bound that applies, computed from the shapes:

* fp64 issue, for the fused kernel: per observation and pass, the D^2 multiply-adds of z @ A, 3 D
  additions and subtractions, and D / 2 Box-Muller pairs of BM_FP64 fp64 instructions each (log,
  sqrt and sincospi, counted in the kernel's SASS), with 2 passes (the second regenerates the row);
  the card does 64 fp64 instructions per clock per SM;
* HBM, for the materialised chain: the data is written once and read twice, n_obs D 8 bytes each,
  at HBM_BYTES_PER_S.

Then the rows/s of the host path (get_model(nd_mean=True).generate: the reference's per-row SciPy
loop) at a size it can finish.  Prints the card's name and power limit first: the numbers belong to
them."""
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from elfi_b200 import ops  # noqa: E402
from elfi_b200.examples import gauss  # noqa: E402

B = 1_000_000
DIMS = (1, 2, 4, 8, 16)
NOBS = (15, 50)
BM_FP64 = 90                 # fp64 instructions per Box-Muller pair (SASS of sim_gauss_nd_kernel)
HBM_BYTES_PER_S = 3.35e12    # H100 SXM5 HBM3


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


def max_clock_hz():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=clocks.max.sm', '--format=csv,noheader,nounits'],
                           capture_output=True, text=True, timeout=30)
        return float(q.stdout.strip().splitlines()[0]) * 1e6
    except (OSError, ValueError, IndexError):
        return 1.98e9


def fp64_bound(D, n_obs, sms, clock):
    per_pass = n_obs * (D * D + 3 * D + D / 2 * BM_FP64)
    return 64 * sms * clock / (2 * per_pass)


def show(label, t, bound, kind):
    rate = B / t[0] * 1e3
    print('  %-44s %8.3f ms (min %.3f, max %.3f)  %.3g rows/s  (%s bound %.3g rows/s, %.0f%%)' % (
        label, *t, rate, kind, bound, 100 * rate / bound))


if not torch.cuda.is_available():
    sys.exit('time_gauss_nd.py measures on a GPU; none is available')
print('card:', card())
sms = torch.cuda.get_device_properties(0).multi_processor_count
clock = max_clock_hz()
rs = np.random.RandomState(0)
for D in DIMS:
    C = rs.randn(D, D) * 0.3
    A = ops.gauss_nd_factor(C @ C.T + np.eye(D), D)
    mu = torch.from_numpy(rs.uniform(-1, 9, (B, D))).cuda()
    for n_obs in NOBS:
        print('D = %d, n_obs = %d, B = %.0e' % (D, n_obs, B))
        show('fused sim_gauss_nd (summaries, no data)',
             timeit(lambda: ops.sim_gauss_nd(mu, A, n_obs, seed=1)),
             fp64_bound(D, n_obs, sms, clock), 'fp64')
        hbm = HBM_BYTES_PER_S / (3 * n_obs * D * 8)
        show('sim_gauss_nd writing Y, then summaries',
             timeit(lambda: ops.gauss_nd_summaries(ops.sim_gauss_nd(
                 mu, A, n_obs, seed=1, want_data=True, want_summaries=False)[0])), hbm, 'HBM')
        Y = ops.sim_gauss_nd(mu, A, n_obs, seed=1, want_data=True, want_summaries=False)[0]
        show('gauss_nd_summaries of Y alone', timeit(lambda: ops.gauss_nd_summaries(Y)),
             HBM_BYTES_PER_S / (2 * n_obs * D * 8), 'HBM')
        del Y
    del mu
    torch.cuda.empty_cache()

for D in (2, 16):
    cov = np.eye(D) + 0.5 * (1 - np.eye(D)) if D == 2 else None
    m = gauss.get_model(true_params=[4] * D, nd_mean=True, cov_matrix=cov, seed_obs=1)
    m.generate(100, outputs=['d'], seed=2)
    Bh = 20_000
    t0 = time.perf_counter()
    m.generate(Bh, outputs=['d'], seed=3)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    print('host gauss.get_model(nd_mean=True), D = %d, n_obs = 50: generate(%d, outputs=[\'d\']) '
          '%.3f s, %.3g rows/s' % (D, Bh, dt, Bh / dt))
