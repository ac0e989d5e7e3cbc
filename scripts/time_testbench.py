#!/usr/bin/env python
"""Timings of the Testbench (elfi_b200/testbench.py) and its two segmented kernels.

* Whole-testbench wall time of one Rejection method (n_samples = 1000, quantile = 0.01) on the
  device MA2 model, serial (run(lockstep=False)) against lock-step (run()), for R repetitions in
  {1, 8, 64} and batch_size in {1e4, 1e5}; one warm-up run per configuration, then the median of
  three, each ending in a device synchronise.  The two runs' samples are compared bit for bit.
* CUDA-event times of ops.dist_seg against R separate ops.dist_euclid calls, and of
  ops.merge_topn_seg against R separate ops.merge_topn calls (n = 1000 kept rows, the distance and
  two parameter outputs, the shapes of one lock-step MA2 batch).
Prints the card's name and power limit first: the numbers belong to them."""
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
from elfi_b200.examples import ma2  # noqa: E402


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                            '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        return q.stdout.strip() or torch.cuda.get_device_name(0)
    except OSError:
        return torch.cuda.get_device_name(0) + ' (power limit not read)'


def device_ms(fn, reps=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(5):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) / reps)
    return float(np.median(ts))


def testbench_run(model, R, batch_size, lockstep):
    tb = elfi.Testbench(model=model, repetitions=R, seed=5, progress_bar=False)
    m = elfi.TestbenchMethod(method=elfi.Rejection)
    m.set_method_kwargs(discrepancy_name='d', batch_size=batch_size)
    m.set_sample_kwargs(n_samples=1000, quantile=0.01, bar=False)
    tb.add_method(m)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    tb.run(lockstep=lockstep)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, tb.testbench_results[0]['results']


def wall_rows():
    model = ma2.get_device_model(seed_obs=4)
    rows = []
    for R in (1, 8, 64):
        for bs in (10000, 100000):
            times = {True: [], False: []}
            res = {}
            for lockstep in (False, True):
                testbench_run(model, R, bs, lockstep)                 # warm-up
            for _ in range(3):
                for lockstep in (False, True):                        # alternated
                    t, res[lockstep] = testbench_run(model, R, bs, lockstep)
                    times[lockstep].append(t)
            same = all(np.array_equal(np.asarray(a.outputs[k]), np.asarray(b.outputs[k]))
                       for a, b in zip(res[True], res[False]) for k in a.outputs)
            row = dict(R=R, batch_size=bs, serial_s=float(np.median(times[False])),
                       lockstep_s=float(np.median(times[True])), identical=bool(same))
            row['speedup'] = row['serial_s'] / row['lockstep_s']
            print('  testbench R=%3d batch=%6d: serial %.4f s, lock-step %.4f s, x%.2f, identical=%s'
                  % (R, bs, row['serial_s'], row['lockstep_s'], row['speedup'], same))
            rows.append(row)
    return rows


def kernel_rows():
    rows = []
    g = torch.Generator(device='cuda').manual_seed(0)
    for R in (8, 64):
        for B in (10000, 100000):
            for D in (2, 128):
                if D == 128 and R * B > 1_000_000:
                    continue
                S = torch.randn(R * B, D, dtype=torch.float64, device='cuda', generator=g)
                obs = torch.randn(R, D, dtype=torch.float64, device='cuda', generator=g)
                seg = device_ms(lambda: ops.dist_seg(S, obs))
                sep = device_ms(lambda: [ops.dist_euclid(S[r * B:(r + 1) * B], obs[r])
                                         for r in range(R)])
                print('  dist   R=%2d B=%6d D=%3d: segmented %.4f ms, %d calls %.4f ms, x%.2f'
                      % (R, B, D, seg, R, sep, sep / seg))
                rows.append(dict(kernel='dist', R=R, B=B, D=D, seg_ms=seg, separate_ms=sep))
            n = 1000
            A = [torch.randn(R, n, dtype=torch.float64, device='cuda', generator=g)
                 for _ in range(3)]
            A[0] = A[0].abs().sort(dim=1).values
            Bs = [torch.randn(R, B, dtype=torch.float64, device='cuda', generator=g).abs()
                  for _ in range(3)]
            seg = device_ms(lambda: ops.merge_topn_seg(A, Bs, A[0], Bs[0], n))
            sep = device_ms(lambda: [ops.merge_topn([a[r] for a in A], [b[r] for b in Bs], A[0][r],
                                                    Bs[0][r], None, n) for r in range(R)])
            print('  merge  R=%2d B=%6d n=%d, 3 outputs: segmented %.4f ms, %d calls %.4f ms, x%.2f'
                  % (R, B, n, seg, R, sep, sep / seg))
            rows.append(dict(kernel='merge', R=R, B=B, n=n, seg_ms=seg, separate_ms=sep))
    return rows


def main():
    torch.cuda.set_device(0)
    c = card()
    print('card:', c)
    kernel_rows()
    wall_rows()


if __name__ == '__main__':
    main()
