#!/usr/bin/env python
"""Timings of lock-step BSL chains (elfi_b200/bsl.py, elfi_b200/csrc/bsl_chains.cu).

* Wall time per iteration and chain-iterations per second on MA2 (n_obs = 50, the series as the
  d = 50 features, n_sim_round = 500) for C in {1, 8, 64, 256} chains:
  parity mode on the device model (host proposals, one likelihood call with G = C per iteration),
  throughput mode on the device model with uniform priors (ops.bsl_mh_step, no per-iteration read).
* Device-to-host copies per iteration, from torch.profiler runs of 10 and 20 iterations (the
  difference divided by 10, so the reads before the first and after the last iteration cancel).
Prints the card's name and power limit first: the numbers belong to them."""
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from elfi_b200 import bsl  # noqa: E402
from elfi_b200.examples import ma2  # noqa: E402

SIGMA = np.array([[.02, .01], [.01, .02]])
CHAINS = (1, 8, 64, 256)


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                            '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        return q.stdout.strip() or torch.cuda.get_device_name(0)
    except OSError:
        return torch.cuda.get_device_name(0) + ' (power limit not read)'


def run(mode, C, iters, seed=123):
    if mode == 'parity':
        m, dp = ma2.get_device_model(n_obs=50, seed_obs=4), None
    else:
        m, dp = ma2.get_uniform_device_model(n_obs=50, seed_obs=4)
    sampler = bsl.BSL(m, 500, ['MA2'], seed=seed, device_proposal=dp)
    return sampler.sample(iters, SIGMA, params0=np.array([.6, .2]), n_chains=C)


def ms_per_iteration(mode, C, iters):
    run(mode, C, 5)                                     # warm-up
    ts = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        run(mode, C, iters)
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3 / iters)
    return float(np.median(ts)), float(min(ts)), float(max(ts))


def d2h_count(mode, C, iters):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        run(mode, C, iters)
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if 'Memcpy DtoH' in e.name)


def main():
    torch.cuda.set_device(0)
    print('card:', card())
    print('BSL on MA2 (n_obs = 50, d = 50, n_sim_round = 500); wall time per iteration, median '
          '(min, max) of 3 runs:')
    for mode in ('parity', 'throughput'):
        for C in CHAINS:
            iters = 100 if C <= 64 else 40
            ms = ms_per_iteration(mode, C, iters)
            d2h = (d2h_count(mode, C, 20) - d2h_count(mode, C, 10)) / 10
            print('  %-10s C = %3d: %8.3f ms per iteration (%.3f, %.3f), %9.0f chain-iterations/s,'
                  ' %.2f device-to-host copies per iteration' % (
                      mode, C, ms[0], ms[1], ms[2], C * 1e3 / ms[0], d2h))


if __name__ == '__main__':
    main()
