#!/usr/bin/env python
"""Timings of Bayesian synthetic likelihood (elfi_b200/csrc/synlik.cu, elfi_b200/bsl.py).

* ops.synlik with CUDA events after warm-up at (G, n, d) = (1, 500, 50), the MA2 BSL round;
  (1, 5000, 145), the scratch assay; (10, 100, 50) with K = 30 penalties, select_penalty.  Next to
  each, the host computation of the reference's gaussian_syn_likelihood on the same inputs
  (np.cov, the Warton shrinkage, scipy.stats.multivariate_normal.logpdf), one call per group and
  penalty.
* Wall time per BSL iteration on MA2 (n_obs = 50, n_sim_round = 500), the device model against
  the host model (host simulator, device likelihood).
* Device-to-host copies per BSL round, counted in a torch.profiler run of its own.
Prints the card's name and power limit first: the numbers belong to them."""
import os
import subprocess
import sys
import time

import numpy as np
import scipy.stats as ss
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from elfi_b200 import bsl, ops  # noqa: E402
from elfi_b200.examples import ma2  # noqa: E402

SIGMA = np.array([[.02, .01], [.01, .02]])


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                            '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        return q.stdout.strip() or torch.cuda.get_device_name(0)
    except OSError:
        return torch.cuda.get_device_name(0) + ' (power limit not read)'


def device_ms(fn, reps=50, warm=5):
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


def host_ms(fn, reps=3):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def host_likelihood(S, y, penalties):
    """The reference's gaussian_syn_likelihood arithmetic per group and penalty."""
    out = []
    for X in S:
        mean, cov = X.mean(0), np.atleast_2d(np.cov(X, rowvar=False))
        for lam in penalties if penalties is not None else [None]:
            c = cov if lam is None else (1 - lam) * cov + lam * np.diag(np.diag(cov) + 1e-5)
            out.append(ss.multivariate_normal.logpdf(y, mean=mean, cov=c))
    return out


def synlik_rows():
    rs = np.random.RandomState(0)
    for G, n, d, K, what in [(1, 500, 50, 0, 'MA2 BSL round'), (1, 5000, 145, 0, 'scratch assay'),
                             (10, 100, 50, 30, 'select_penalty')]:
        A = np.eye(d) + 0.3 * rs.randn(d, d) / np.sqrt(d)
        S = rs.randn(G, n, d) @ A
        y = S[0].mean(0) + 0.1 * rs.randn(d)
        pens = np.linspace(0.2, 0.78, K) if K else None
        Sd = torch.from_numpy(S).cuda()
        yd = torch.from_numpy(y).cuda()
        t = device_ms(lambda: ops.synlik(Sd, yd, penalties=pens))
        h = host_ms(lambda: host_likelihood(S, y, pens))
        print('  synlik (G, n, d) = (%d, %d, %d), K = %d [%s]: device %.4f ms (min %.4f, max %.4f);'
              ' host NumPy/SciPy %.3f ms; ratio %.0f' % (G, n, d, K, what, *t, h, h / t[0]))


def bsl_iteration_ms(model, iters):
    sampler = bsl.BSL(model, 500, ['MA2'], seed=123)
    sampler.sample(10, sigma_proposals=SIGMA, params0=np.array([.6, .2]))     # warm-up
    sampler = bsl.BSL(model, 500, ['MA2'], seed=123)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = sampler.sample(iters, sigma_proposals=SIGMA, params0=np.array([.6, .2]))
    torch.cuda.synchronize()
    rounds = res.n_sim // 500
    return (time.perf_counter() - t0) * 1e3 / iters, rounds


def d2h_per_round(model, iters=20):
    from torch.profiler import ProfilerActivity, profile
    bsl.BSL(model, 500, ['MA2'], seed=7).sample(5, sigma_proposals=SIGMA,
                                                params0=np.array([.6, .2]))
    sampler = bsl.BSL(model, 500, ['MA2'], seed=7)
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        res = sampler.sample(iters, sigma_proposals=SIGMA, params0=np.array([.6, .2]))
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    d2h = sum(1 for nm in names if 'Memcpy DtoH' in nm)
    kernels = sum(1 for nm in names if 'synlik_factor_kernel' in nm)
    return d2h, res.n_sim // 500, kernels


def main():
    torch.cuda.set_device(0)
    print('card:', card())
    print('ops.synlik (CUDA events, median of 5 windows of 50 calls):')
    synlik_rows()
    dev_model = ma2.get_device_model(n_obs=50, seed_obs=4)
    host_model = ma2.get_model(n_obs=50, true_params=[.6, .2], seed_obs=4)
    for label, m in [('device model', dev_model), ('host model', host_model)]:
        ms, rounds = bsl_iteration_ms(m, 200)
        print('  BSL on MA2, %s: %.3f ms per iteration (200 iterations, %d simulated rounds)' % (
            label, ms, rounds))
    d2h, rounds, kernels = d2h_per_round(dev_model)
    print('  profiler, device model: %d device-to-host copies over %d simulated rounds (%.2f per '
          'round), %d likelihood factor kernels' % (d2h, rounds, d2h / max(rounds, 1), kernels))


if __name__ == '__main__':
    main()
