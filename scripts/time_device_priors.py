#!/usr/bin/env python
"""CUDA-event timings of the stock-prior kernels (elfi_b200/csrc/prior.cu) and of the mixture
proposals with support 3, plus one SMC population of a six-parameter model with device against host
priors and proposals.  Prints the card's name and power limit first: the numbers belong to them."""
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import elfi_b200 as elfi  # noqa: E402
from elfi_b200 import ops  # noqa: E402
from elfi_b200.priors import prior_spec  # noqa: E402


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
    return float(np.median(ts)), float(min(ts)), float(max(ts))


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                            '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        return q.stdout.strip() or torch.cuda.get_device_name(0)
    except OSError:
        return torch.cuda.get_device_name(0) + ' (power limit not read)'


print('card:', card())
B = 1_000_000
for kind, params in [('uniform', (0.0, 10.0)), ('norm', (50.0, 7.0)), ('truncnorm', (0.0, 5.0)),
                     ('expon', (np.e, 2.0)), ('gamma', (0.3,)), ('gamma', (2.5,)),
                     ('beta', (0.5, 0.5)), ('beta', (2.0, 5.0))]:
    spec = prior_spec(kind, params)
    med, lo, hi = timeit(lambda: ops.prior_rvs(spec, B, seed=1))
    print('prior_rvs %-9s %-16s B=1e6: %.4f ms (min %.4f, max %.4f), %.1f GB/s of output'
          % (kind, params, med, lo, hi, 8 * B / med / 1e6))

rs = np.random.RandomState(0)
N = 10000
for p in (4, 8, 16):
    means = rs.uniform(1, 9, (N, p))
    cov = np.eye(p) * 0.5
    cdf = ops.gm_cdf(rs.rand(N), N)
    mdev = torch.from_numpy(means).cuda()
    specs = np.array([prior_spec('uniform', (0.0, 10.0))] * p)
    box = ([0.0] * p, [10.0] * p)
    rows = []
    for support in (2, 3):
        kw = dict(box=box) if support == 2 else dict(prior=specs)
        med, lo, hi = timeit(lambda: ops.gm_rvs(mdev, cov, None, B, seed=3, support=support, cdf=cdf, **kw))
        rows.append('support %d: %.3f ms (min %.3f, max %.3f)' % (support, med, lo, hi))
    print('gm_rvs p=%2d uniform(0, 10) priors, N=1e4, B=1e6: %s' % (p, '; '.join(rows)))

# one SMC population of the six-parameter model: device priors + proposals vs host
import device_prior_cases as cases  # noqa: E402

m = cases.six_model()
dp = elfi.DeviceModelPrior(m)
def smc_seconds(model, quantiles, **kw):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    elfi.SMC(model['d'], batch_size=100000, seed=5, **kw).sample(10000, quantiles=quantiles, bar=False)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


for label, model, kw in (('device', dp.model, dict(device_proposal=dp)), ('host', m, {})):
    smc_seconds(model, [0.1, 0.3], **kw)                       # warm-up
    one = [smc_seconds(model, [0.1], **kw) for _ in range(3)]
    two = [smc_seconds(model, [0.1, 0.3], **kw) for _ in range(3)]
    print('SMC, six-parameter model, 10000 particles, batches of 1e5, %s priors and proposals: '
          'round 0 alone %.3f s, rounds 0 + 1 %.3f s (medians of 3) -> one proposal population '
          '%.3f s' % (label, np.median(one), np.median(two), np.median(two) - np.median(one)))
