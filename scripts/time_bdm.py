#!/usr/bin/env python
"""CUDA-event timings of the birth-death-mutation kernels (elfi_b200/csrc/bdm.cu): ops.sim_bdm at
B = 1e6 prior draws (alpha ~ U(0.005, 2.005), delta = 0, tau = 0.198) for N = 20 and for N = 473
(Tanaka's San Francisco data), with the events per second; the share of the fused T1 / T2 (the
simulator with summaries against the simulator writing only the counts); a throughput-mode
Rejection on get_device_model(); then the rows/s of the host path through the reference's
executable, when oracle/_ref/bdm exists.  Prints the card's name and power limit first: the
numbers belong to them.  Fails without a GPU."""
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import elfi_b200 as elfi  # noqa: E402
from elfi_b200 import ops  # noqa: E402
from elfi_b200.examples import bdm  # noqa: E402

EXE = os.path.join(ROOT, 'oracle', '_ref', 'bdm')


def timeit(fn, batches=5, warm=1):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(batches):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(min(ts)), float(max(ts))


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                        '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def prior(B, seed):
    rs = np.random.RandomState(seed)
    return np.column_stack([rs.uniform(0.005, 2.005, B), np.zeros(B), np.full(B, 0.198)])


if not torch.cuda.is_available():
    raise SystemExit('time_bdm.py needs a CUDA device')
print('card:', card())
B = 1_000_000
for N in (20, 473):
    P = torch.from_numpy(prior(B, 1)).cuda()
    t_s = timeit(lambda: ops.sim_bdm(P, N, seed=1, want_data=False))
    t_x = timeit(lambda: ops.sim_bdm(P, N, seed=1, want_summaries=False))
    n = ops.sim_bdm(P, N, seed=1, want_data=False)[2].cpu().numpy()
    print('N = %d, B = %.0e prior draws: sim_bdm with T1/T2 %.2f ms (min %.2f, max %.2f), %.3g '
          'rows/s, %.3g events/s; counts only %.2f ms (min %.2f, max %.2f); events per row median '
          '%d, max %d, capped %d' % (N, B, *t_s, B / t_s[0] * 1e3, n.sum() / t_s[0] * 1e3, *t_x,
                                     int(np.median(n)), int(n.max()), int((n < 0).sum())))
    X = ops.sim_bdm(P, N, seed=1, want_summaries=False)[0]
    t_u = timeit(lambda: ops.bdm_summaries(X))
    print('N = %d: bdm_summaries of written counts %.3f ms; fused summaries cost %.1f %% of the '
          'simulator (with minus counts-only, over with)'
          % (N, t_u[0], 100.0 * (t_s[0] - t_x[0]) / t_s[0]))
    del P, X
    torch.cuda.empty_cache()

m, _ = bdm.get_device_model()
elfi.Rejection(m['d'], batch_size=1_000_000, seed=1).sample(1000, quantile=0.1, bar=False)
torch.cuda.synchronize()
t0 = time.perf_counter()
res = elfi.Rejection(m['d'], batch_size=1_000_000, seed=2).sample(100_000, quantile=0.1, bar=False)
torch.cuda.synchronize()
dt = time.perf_counter() - t0
print('throughput-mode Rejection on get_device_model(), %d simulations (100000 accepted): '
      '%.3f s, %.3g simulations/s' % (res.n_sim, dt, res.n_sim / dt))

if os.path.isfile(EXE):
    work = tempfile.mkdtemp()
    cwd = os.getcwd()
    try:
        shutil.copy(EXE, os.path.join(work, 'bdm'))
        os.chdir(work)
        for N in (20, 473):
            n_host = 20_000 if N == 20 else 2_000
            meta = dict(model_name='bdm', batch_index=0, submission_index=0)
            a = prior(n_host, 2)[:, 0]
            t0 = time.perf_counter()
            bdm.BDM(a, 0.0, 0.198, N, random_state=np.random.RandomState(0), meta=meta)
            dt = time.perf_counter() - t0
            print('host path (executable, input and output files), N = %d, B = %d: %.3f s, %.3g '
                  'rows/s' % (N, n_host, dt, n_host / dt))
    finally:
        os.chdir(cwd)
        shutil.rmtree(work)
else:
    print('host path: oracle/_ref/bdm absent, not timed')
