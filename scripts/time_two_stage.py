"""Time TwoStageSelection on the device MA2 model: the all-combination device path against the
per-combination rejection loop, each new kernel with CUDA events, and the device-to-host copies of
one run (counted in a torch.profiler run of its own).

    python scripts/time_two_stage.py [--loop-limit 24]

The loop is timed on at most --loop-limit combinations per configuration; its time per
combination is printed with the number of combinations it was measured on.
"""
import argparse
import os
import subprocess
import sys
import time
from functools import partial
from itertools import combinations

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from elfi_b200 import TwoStageSelection, ops  # noqa: E402
from elfi_b200.examples import gauss, ma2  # noqa: E402
from elfi_b200.throughput import LazySimulation  # noqa: E402

CONFIGS = [(3, 3, 10 ** 5), (8, 3, 10 ** 6), (12, 4, 10 ** 6)]
BATCH = 10 ** 5


def named(fn, name):
    fn.__name__ = name
    return fn


def materialised(stat, name):
    return named(lambda y: stat(y.materialize() if isinstance(y, LazySimulation) else y), name)


def candidates(n):
    """ac_lag1 and ac_lag2 from the simulator kernel, the mean, the variance, then further lags."""
    out = [named(partial(ma2.autocov, lag=1), 'ac1'), named(partial(ma2.autocov, lag=2), 'ac2'),
           materialised(gauss.ss_mean, 'mean'), materialised(gauss.ss_var, 'var')]
    lag = 3
    while len(out) < n:
        out.append(materialised(partial(ma2.autocov, lag=lag), 'ac{}'.format(lag)))
        lag += 1
    return out[:n]


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                        '--format=csv,noheader'], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def events(fn, reps=20):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--loop-limit', type=int, default=24)
    args = ap.parse_args()
    print('card: {}'.format(card()))
    model = ma2.get_device_model(seed_obs=0)
    sim = model['MA2']
    for n_cand, cardinality, n_sim in CONFIGS:
        sel = TwoStageSelection(sim, 'euclidean', list_ss=candidates(n_cand),
                                max_cardinality=cardinality, seed=0)
        C = len(sel.ss_candidates)
        sel.run(n_sim=min(n_sim, 2 * BATCH), batch_size=BATCH)      # warm-up
        t_dev, chosen = wall(lambda: sel.run(n_sim=n_sim, batch_size=BATCH))
        n_acc = int(n_sim / 100)
        m = min(C, args.loop_limit)
        t_loop, _ = wall(lambda: [sel._obtain_accepted_thetas(s, n_sim, n_acc, BATCH)
                                  for s in sel.ss_candidates[:m]])
        print('candidates={} cardinality={} combinations={} n_sim={}: device path {:.3f} s; '
              'rejection loop {:.3f} s per combination (timed on {} of {}), {:.1f} s for all '
              'by that rate; selected {}'.format(n_cand, cardinality, C, n_sim, t_dev, t_loop / m,
                                                 m, C, t_loop / m * C,
                                                 [f.__name__ for f in chosen]))

    # kernels at the largest configuration's shapes: TwoStageSelection scores combinations in
    # groups whose (group x n_sim) distance block fits its 256 MiB budget
    rs = np.random.RandomState(0)
    combs = [[(j, 1) for j in c] for r in range(1, 5) for c in combinations(range(12), r)]
    rows = 10 ** 6
    C = (256 << 20) // (8 * rows)
    S = torch.tensor(rs.randn(rows, 12), device='cuda')
    obs = rs.randn(12)
    layout = ops.SubsetLayout(combs[-C:], 12)
    out = torch.empty((C, rows), dtype=torch.float64, device='cuda')
    ms = events(lambda: ops.subset_distance(S, obs, layout, 'euclidean', out=out))
    print('subset_distance: C={} of cardinality 4, rows={} W=12: {:.3f} ms ({:.1f} GB/s of summary rows and '
          'distances)'.format(C, rows, ms, (S.numel() + out.numel()) * 8 / ms / 1e6))
    for n in (1000, 10000):
        X = torch.tensor(rs.randn(C, n, 2), device='cuda')
        ms = events(lambda: ops.knn_entropy(X, 4), reps=3)
        print('knn_entropy: C={} n={} q=2 k=4: {:.3f} ms ({:.2f} G pairs/s)'.format(
            C, n, ms, C * n * n / ms / 1e6))
        P = X[0, :n // 100]
        ms = events(lambda: ops.mrsse(X, P), reps=5)
        print('mrsse: C={} n={} q=2 m={}: {:.3f} ms'.format(C, n, n // 100, ms))

    # device-to-host copies of one run
    sel = TwoStageSelection(sim, 'euclidean', list_ss=candidates(8), max_cardinality=3, seed=0)
    sel.run(n_sim=2 * BATCH, batch_size=BATCH)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        sel.run(n_sim=10 ** 6, batch_size=BATCH)
        torch.cuda.synchronize()
    d2h = [e for e in prof.events() if 'DtoH' in e.name or 'Device -> Host' in e.name]
    print('device-to-host copies in one run (8 candidates, cardinality 3, n_sim=1e6): {}'.format(
        len(d2h)))


if __name__ == '__main__':
    main()
