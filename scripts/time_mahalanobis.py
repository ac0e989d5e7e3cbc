#!/usr/bin/env python
"""Timings of the Mahalanobis distance (elfi_b200_dist_mahalanobis_thr_f64, elfi_b200/csrc/distance.cu).

* ops.dist_mahalanobis with CUDA events after warm-up, at B in {1e5, 1e6} and D in {2, 16, 50, 145},
  rows, obs and VI already on the device and no threshold.  Next to each, ops.dist_seuclidean at the
  same shape (the other distance with a matrix-free keyword, one pass over the row) and host
  scipy.spatial.distance.cdist(..., 'mahalanobis', VI=VI).  The host time is measured on the first
  HOST_ROWS rows and scaled to B: cdist's loop is linear in the rows.
* Work from the shapes: per row 2 D^2 + 2 D fp64 operations (t = VI u and u . t, each product and
  sum its own instruction: no FMA, which bit-identity with SciPy rules out) and 8 D bytes read +
  8 bytes written.  The bound that applies is the larger of operations / fp64 issue rate and
  bytes / HBM bandwidth, both from NVIDIA's H100 SXM data sheet at 700 W: 34 TFLOP/s fp64 (an FMA
  counted as two operations, so 17e12 unfused operations per second) and 3.35 TB/s.  The share is
  that bound over the measured time.
Prints the card's name and power limit first: the numbers belong to them."""
import os
import subprocess
import sys
import time

import numpy as np
import torch
from scipy.spatial.distance import cdist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from elfi_b200 import ops  # noqa: E402

FP64_UNFUSED_OPS = 34e12 / 2   # data sheet fp64 (non-tensor) rate, an FMA counted as two
HBM_BYTES = 3.35e12
HOST_ROWS = 20000


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
    return float(np.median(ts)), float(min(ts)), float(max(ts))


def host_ms(fn):
    fn()
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3


def row(B, D, rs):
    A = rs.randn(D, D)
    VI = A @ A.T / D + np.eye(D)
    obs = rs.randn(D)
    S = torch.randn(B, D, dtype=torch.float64, device='cuda')
    S_host = S[:HOST_ROWS].cpu().numpy()
    VI_d, obs_d = torch.from_numpy(VI).cuda(), torch.from_numpy(obs).cuda()
    V_d = torch.from_numpy(1.0 / np.diag(VI)).cuda()
    t = device_ms(lambda: ops.dist_mahalanobis(S, obs_d, VI_d))
    ts = device_ms(lambda: ops.dist_seuclidean(S, obs_d, V_d))
    h = host_ms(lambda: cdist(S_host, obs[None], 'mahalanobis', VI=VI)) * B / len(S_host)
    ops_n = B * (2.0 * D * D + 2.0 * D)
    bytes_n = B * (8.0 * D + 8.0)
    t_ops, t_bytes = ops_n / FP64_UNFUSED_OPS, bytes_n / HBM_BYTES
    bound, which = (t_ops, 'fp64 issue') if t_ops >= t_bytes else (t_bytes, 'HBM')
    sec = t[0] * 1e-3
    print('  B=%-8d D=%-4d mahalanobis %9.4f ms (min %.4f, max %.4f)  %6.2f Tops/s  %7.1f GB/s  '
          '%5.1f%% of the %s bound | seuclidean %8.4f ms | host cdist %10.1f ms (x%.0f)' % (
              B, D, *t, ops_n / sec * 1e-12, bytes_n / sec * 1e-9, 100 * bound / sec, which,
              ts[0], h, h / t[0]))
    del S


def main():
    torch.cuda.set_device(0)
    print('card:', card())
    print('ops.dist_mahalanobis (CUDA events after warm-up, median of 5 windows of 20 calls; '
          'host cdist on %d rows, scaled to B):' % HOST_ROWS)
    rs = np.random.RandomState(0)
    torch.manual_seed(0)
    for B in (100000, 1000000):
        for D in (2, 16, 50, 145):
            row(B, D, rs)


if __name__ == '__main__':
    main()
