#!/usr/bin/env python
"""Timings of Wood's 13 Ricker statistics (elfi_b200/csrc/ricker_wood.cu): CUDA-event time of
ops.wood_summaries on device-simulated counts at n_obs = 50 and 500 for B = 1e5 and 1e6, the rows/s
of the host NumPy definition (ricker.wood_statistics) at B = 1e4, and one throughput-mode BSL
iteration on get_device_model(summary='wood') at n_sim_round = 500 for 1 and 64 chains.  Prints the
card's name and power limit first: the numbers belong to them."""
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from elfi_b200 import bsl, ops  # noqa: E402
from elfi_b200.examples import ricker  # noqa: E402

TRUTH = (3.8, 0.3, 10.0)


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


def show(label, t, rows):
    print('  %-44s %9.3f ms (min %.3f, max %.3f)  %.3g rows/s' % (label, *t, rows / t[0] * 1e3))


print('card:', card())
for n_obs in (50, 500):
    obs = ricker.stochastic_ricker(*TRUTH, n_obs=n_obs, random_state=np.random.RandomState(1))
    P = torch.from_numpy(ricker.wood_design(obs)).cuda()
    for B in (100_000, 1_000_000):
        Y = ops.sim_ricker(np.tile(TRUTH, (B, 1)), n_obs, seed=2, want_data=True,
                           want_summaries=False)[0]
        show('wood_summaries, n_obs = %d, B = %.0e' % (n_obs, B),
             timeit(lambda: ops.wood_summaries(Y, P)), B)
        del Y
        torch.cuda.empty_cache()
    y = ricker.stochastic_ricker(*TRUTH, n_obs=n_obs, batch_size=10_000,
                                 random_state=np.random.RandomState(3))
    design = ricker.wood_design(obs)
    ricker.wood_statistics(y, design)
    t0 = time.perf_counter()
    for _ in range(3):
        ricker.wood_statistics(y, design)
    dt = (time.perf_counter() - t0) / 3
    print('  %-44s %9.3f ms  %.3g rows/s' % ('host NumPy definition, n_obs = %d, B = 1e4' % n_obs,
                                             dt * 1e3, 1e4 / dt))

# one BSL iteration in throughput mode: simulation, statistics, likelihood and the device MH step
m = ricker.get_model(n_obs=50, seed_obs=2, summary='wood')
pilot = m.generate(2000, ['Wood'], with_values=dict(zip(['t1', 't2', 't3'], TRUTH)), seed=1)['Wood']
lik = bsl.standard_likelihood(whitening=np.diag(1 / np.std(pilot, axis=0)))
dm, dp = ricker.get_device_model(n_obs=50, seed_obs=2, summary='wood')
sigma = np.diag([0.01, 0.004, 0.25])
for chains in (1, 64):
    params0 = np.tile(TRUTH, (chains, 1)) if chains > 1 else np.array(TRUTH)

    def run(n_iter, seed):
        s = bsl.BSL(dm, 500, ['Wood'], likelihood=lik, seed=seed, device_proposal=dp)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        s.sample(n_iter, sigma, params0=params0, n_chains=chains)
        torch.cuda.synchronize()
        return time.perf_counter() - t0
    run(20, 1)
    short, long_ = run(50, 2), run(250, 3)
    per = (long_ - short) / 200
    print('  throughput BSL, n_obs = 50, n_sim_round = 500, %2d chain(s): %.3f ms per iteration '
          '(%.3g simulations/s)' % (chains, per * 1e3, chains * 500 / per))
