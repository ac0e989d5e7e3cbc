"""Time ROMC per phase with CUDA events: the device MA2 model at n1 in {1e3, 1e4, 1e5} (solve,
Hessian, regions, surrogates, sample, a 1e5-point posterior grid) and the host MA2 model at
n1 = 100.  Prints the card's name and power limit with the numbers, one JSON line per run.

    python scripts/time_romc.py [--n1 1000 10000 100000] [--host-n1 100]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from elfi_b200 import romc  # noqa: E402
from elfi_b200.examples import ma2  # noqa: E402


def card():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else torch.cuda.get_device_name(0)


def phase(times, name, fn):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    start.record()
    out = fn()
    end.record()
    torch.cuda.synchronize()
    times[name] = {'event_ms': start.elapsed_time(end), 'wall_ms': 1e3 * (time.perf_counter() - t0)}
    return out


def run(model, n1, device_prior, grid):
    r = romc.ROMC(model['d'], [(-2, 2), (-1, 1)], device_prior=device_prior)
    t = {}
    phase(t, 'solve+hessian', lambda: r.solve_problems(n1=n1, seed=1))
    eps = float(r.compute_eps(0.3))
    phase(t, 'regions', lambda: r.estimate_regions(eps, fit_models=False))
    phase(t, 'regions+surrogates', lambda: r.estimate_regions(eps, fit_models=True))
    phase(t, 'sample', lambda: r.sample(n2=50, seed=2))
    if grid:
        g = np.random.RandomState(0).uniform([-2, -1], [2, 1], (100000, 2))
        phase(t, 'posterior_grid_1e5', lambda: r.eval_unnorm_posterior(g))
    return {'n1': n1, 'regions': int(len(r.center)), 'mean_nfev': float(np.mean(r.nfev)),
            'times': t}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n1', type=int, nargs='+', default=[1000, 10000, 100000])
    ap.add_argument('--host-n1', type=int, default=100)
    a = ap.parse_args()
    name = card()
    dm = ma2.get_device_model(n_obs=100, true_params=[.6, .2], seed_obs=4)
    run(dm, 200, ma2.DeviceProposal, False)               # warm-up of every shape's kernels
    for n1 in a.n1:
        print(json.dumps({'card': name, 'model': 'MA2 device', **run(dm, n1, ma2.DeviceProposal,
                                                                    True)}))
    if a.host_n1:
        hm = ma2.get_model(n_obs=100, true_params=[.6, .2], seed_obs=4)
        print(json.dumps({'card': name, 'model': 'MA2 host', **run(hm, a.host_n1, None, False)}))


if __name__ == '__main__':
    main()
