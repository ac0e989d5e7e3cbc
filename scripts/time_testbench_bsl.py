#!/usr/bin/env python
"""Timings of a whole Testbench with one BSL method (elfi_b200/testbench.py, lock-step BSL).

MA2 with n_obs = 50 and the series as the d = 50 features, n_sim_round = 500, 200 iterations, for
R in {1, 8, 32} repetitions:
* parity mode on ma2.get_device_model() (host proposals and decisions);
* throughput mode on ma2.get_uniform_device_model() with device_proposal (the device prior table
  does not cover MA2's triangular prior; the uniform box around it does).
Serial (run(lockstep=False)) and lock-step (run()) alternate, after one warm-up run of each; the
median of three timed runs, each ending in a device synchronise.  The two paths' samples and
n_sim are compared bit for bit.  Prints the card's name and power limit first: the numbers belong
to them.  Writes nothing."""
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import elfi_b200 as elfi  # noqa: E402
from elfi_b200 import bsl  # noqa: E402
from elfi_b200.examples import ma2  # noqa: E402

REPS = (1, 8, 32)
N_ITER = 200
SIGMA = np.array([[.02, .01], [.01, .02]])


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                            '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        return q.stdout.strip() or torch.cuda.get_device_name(0)
    except OSError:
        return torch.cuda.get_device_name(0) + ' (power limit not read)'


def models():
    dm = ma2.get_device_model(n_obs=50, true_params=[.6, .2], seed_obs=4)
    um, dp = ma2.get_uniform_device_model(n_obs=50, true_params=[.6, .2], seed_obs=4)
    return {'parity': (dm, {}), 'throughput': (um, dict(device_proposal=dp))}


def run(model, mk, R, lockstep):
    tb = elfi.Testbench(model=model, repetitions=R, seed=156, progress_bar=False)
    m = elfi.TestbenchMethod(method=bsl.BSL, name='BSL')
    m.set_method_kwargs(n_sim_round=500, feature_names=['MA2'], **mk)
    m.set_sample_kwargs(n_samples=N_ITER, sigma_proposals=SIGMA, params0=np.array([.6, .2]))
    tb.add_method(m)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    tb.run(lockstep=lockstep)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, tb.testbench_results[0]['results']


def same(a, b):
    return all(np.array_equal(s.samples_all[k], t.samples_all[k]) and s.n_sim == t.n_sim
               and s.acc_rate == t.acc_rate for s, t in zip(a, b) for k in s.samples_all)


def main():
    torch.cuda.init()
    print('card:', card())
    print('whole testbench, BSL on MA2 (n_obs = 50, d = 50, n_sim_round = 500, {} iterations); '
          'median of 3 alternated runs after warm-up'.format(N_ITER))
    print('| mode | R | serial | lock-step | speed-up | identical |')
    print('|---|---|---|---|---|---|')
    for mode, (model, mk) in models().items():
        for R in REPS:
            run(model, mk, R, False)
            run(model, mk, R, True)
            ts = {False: [], True: []}
            res = {}
            for _ in range(3):
                for lockstep in (False, True):
                    t, res[lockstep] = run(model, mk, R, lockstep)
                    ts[lockstep].append(t)
            serial, lock = np.median(ts[False]), np.median(ts[True])
            print('| {} | {} | {:.3f} s | {:.3f} s | {:.2f}x | {} |'.format(
                mode, R, serial, lock, serial / lock, same(res[True], res[False])), flush=True)


if __name__ == '__main__':
    main()
