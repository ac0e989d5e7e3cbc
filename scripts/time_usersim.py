#!/usr/bin/env python
"""CUDA-event timings of a user-written simulator (tools.cuda_simulator / ops.usersim_run, compiled
at run time by NVRTC) against the built-in kernel it restates: MA(2) as tests/test_usersim_gpu.py
writes it against ops.sim_ma2, at n_obs = 100 and B = 1e6, in rows/s, with the summaries fused
(no data written), with the data written, and with both.  The two kernels are timed alternately,
three rounds.  Then the first compile of a new source and a compile the context has cached, in
seconds.  Prints the card's name and power limit first: the numbers belong to them."""
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from elfi_b200 import ops  # noqa: E402
from test_usersim_gpu import MA2_SALT, MA2_SOURCE  # noqa: E402

N_OBS = 100
B = 1_000_000

# the same MA(2) with the built-in kernel's schedule: four blocks drawn, then eight values written
MA2_EIGHT_SOURCE = r'''
__device__ void simulate(const double* theta, elfi::RowStream& rng, double* y) {
    const double t1 = theta[0], t2 = theta[1];
    double wm2, wm1;
    rng.normal2(0, wm2, wm1);
    for (int k0 = 0; k0 < elfi::n_out; k0 += 8) {
        double w[10];
        w[0] = wm2;
        w[1] = wm1;
#pragma unroll
        for (int q = 0; q < 4; ++q) rng.normal2(1 + k0 / 2 + q, w[2 + 2 * q], w[3 + 2 * q]);
#pragma unroll
        for (int e = 0; e < 8; ++e)
            if (k0 + e < elfi::n_out)
                y[k0 + e] = __dadd_rn(__dadd_rn(w[e + 2], __dmul_rn(t1, w[e + 1])), __dmul_rn(t2, w[e]));
        wm2 = w[8];
        wm1 = w[9];
    }
}
'''


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


def show(label, t):
    print('  %-44s %8.3f ms (min %.3f, max %.3f)  %.3g rows/s' % (label, *t, B / t[0] * 1e3))


if not torch.cuda.is_available():
    sys.exit('time_usersim.py measures on a GPU; none is available')
print('card:', card())
rs = np.random.RandomState(0)
t1 = torch.from_numpy(rs.uniform(-1.5, 1.5, B)).cuda()
t2 = torch.from_numpy(rs.uniform(-0.8, 0.8, B)).cuda()
sim = ops.usersim_compile(MA2_SOURCE, 2, N_OBS, n_summaries=2, salt=MA2_SALT)
cases = [
    ('fused summaries',
     lambda: ops.usersim_run(sim, [t1, t2], seed=1),
     lambda: ops.sim_ma2(t1, t2, N_OBS, seed=1)),
    ('data written',
     lambda: ops.usersim_run(sim, [t1, t2], seed=1, want_data=True, want_summaries=False),
     lambda: ops.sim_ma2(t1, t2, N_OBS, seed=1, want_data=True, want_summaries=False)),
    ('data written and summaries',
     lambda: ops.usersim_run(sim, [t1, t2], seed=1, want_data=True),
     lambda: ops.sim_ma2(t1, t2, N_OBS, seed=1, want_data=True)),
]
eight = ops.usersim_compile(MA2_EIGHT_SOURCE, 2, N_OBS, salt=MA2_SALT)
ye = ops.usersim_run(eight, [t1, t2], seed=1, want_data=True, want_summaries=False)[0]
assert torch.equal(ye, ops.sim_ma2(t1, t2, N_OBS, seed=1, want_data=True, want_summaries=False)[0])
cases.append(('data written, eight values a step',
              lambda: ops.usersim_run(eight, [t1, t2], seed=1, want_data=True, want_summaries=False),
              lambda: ops.sim_ma2(t1, t2, N_OBS, seed=1, want_data=True, want_summaries=False)))
print('MA(2), B = %.0e, n_obs = %d' % (B, N_OBS))
for rnd in range(3):
    print('round', rnd)
    for label, user, builtin in cases:
        show('user    ' + label, timeit(user))
        show('builtin ' + label, timeit(builtin))

# the first compile of a source this process has not seen (a unique comment), then the cached one
source = MA2_SOURCE + '\n// compiled at %r\n' % time.time()
for label in ('first compile', 'cached compile'):
    t0 = time.perf_counter()
    s = ops.usersim_compile(source, 2, N_OBS, n_summaries=2, salt=MA2_SALT)
    dt = time.perf_counter() - t0
    print('%s: %.4f s (NVRTC compilations so far: %d)' % (label, dt, ops.usersim_compiles()))
