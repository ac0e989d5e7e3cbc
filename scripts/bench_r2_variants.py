#!/usr/bin/env python
"""Timings of the row sort, the nested and fused distances and the standardised Euclidean distance
(`WHAT` selects among them).  CUDA events around batches of back-to-back launches."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from elfi_b200 import ops  # noqa: E402

HBM = json.load(open(os.path.join(ROOT, 'MEASURED_PEAKS.json')))['hbm_gbs'] \
    if os.path.exists(os.path.join(ROOT, 'MEASURED_PEAKS.json')) else 6650.0
WHAT = set(os.environ.get('WHAT', 'rowsort,fused,nested,seuclid').split(','))
gen = torch.Generator(device='cuda').manual_seed(0)


def randn(*shape):
    return torch.randn(*shape, dtype=torch.float64, device='cuda', generator=gen)


def timeit(fn, per_batch=10, batches=7, warm=3):
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
    return float(np.median(ts)), float(np.min(ts))


def rec(name, ms, best, nbytes):
    print(json.dumps(dict(name=name, ms_median=round(ms, 4), ms_min=round(best, 4),
                          GBps=round(nbytes / ms / 1e6, 1),
                          frac_hbm_measured=round(nbytes / ms / 1e6 / HBM, 4))), flush=True)


if 'rowsort' in WHAT:
    for B, n in ((1_000_000, 256), (1_000_000, 100), (2_000_000, 50), (250_000, 512)):
        Y = randn(B, n)
        ms, best = timeit(lambda: ops.rowsort(Y), per_batch=3, batches=5, warm=2)
        rec('rowsort {}x{}'.format(B, n), ms, best, 2 * B * n * 8)
        del Y
if 'fused' in WHAT or 'nested' in WHAT:
    B, D = 500_000, 256
    S, obs = randn(B, D), randn(D)
    for K in (2, 5, 6):
        W = torch.rand(K, D, dtype=torch.float64, device='cuda', generator=gen) + 0.5
        Wn = W.cpu().numpy()
        if 'nested' in WHAT:
            ms, best = timeit(lambda: ops.dist_euclid(S, obs, w=Wn))
            rec('nested K={} 5e5x256'.format(K), ms, best, B * D * 8 + B * K * 8)
        if 'fused' in WHAT:
            ms, best = timeit(lambda: ops.dist_euclid(S, obs, w=Wn, moments=True))
            rec('fused K={} + colmoments 5e5x256'.format(K), ms, best, B * D * 8 + B * K * 8)
    del S
if 'seuclid' in WHAT:
    S, obs = randn(1_000_000, 128), randn(128)
    V = np.random.RandomState(0).uniform(0.5, 2.0, 128)
    ms, best = timeit(lambda: ops.dist_seuclidean(S, obs, V))
    rec('seuclidean 1e6x128', ms, best, S.numel() * 8 + S.shape[0] * 8)
    ms, best = timeit(lambda: ops.dist_euclid(S, obs, w=1.0 / V))
    rec('weighted K=1 1e6x128', ms, best, S.numel() * 8 + S.shape[0] * 8)
