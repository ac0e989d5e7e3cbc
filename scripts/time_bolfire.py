#!/usr/bin/env python
"""Timings of BOLFIRE (elfi_b200/csrc/logreg.cu, elfi_b200/bolfire.py).

* ops.logreg_fit + ops.logreg_predict (one query row) with CUDA events after warm-up at (rows per
  class, d) = (500, 17), the ARCH round; (1000, 50); (20000, 160), with the Newton steps taken.
  When scikit-learn imports, the host liblinear fit (StandardScaler + LogisticRegression(penalty=
  'l1', solver='liblinear'), the reference's classifier) on the same problems, labelled host.
* One fully device-side ARCH BOLFIRE round (arch.get_device_model, 500 rows per class), split into
  simulation, classifier (fit, predict and the one read) and GP update + acquisition.
Prints the card's name and power limit first: the numbers belong to them."""
import os
import subprocess
import sys
import time
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from elfi_b200 import bolfire as bf  # noqa: E402
from elfi_b200 import ops  # noqa: E402
from elfi_b200.examples import arch  # noqa: E402


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                            '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        return q.stdout.strip() or torch.cuda.get_device_name(0)
    except OSError:
        return torch.cuda.get_device_name(0) + ' (power limit not read)'


def device_ms(fn, reps=10, warm=2):
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


def problem(n_per, d, seed=0):
    rs = np.random.RandomState(seed)
    X = np.vstack([rs.randn(n_per, d) + 0.3, rs.randn(n_per, d) * 1.3])
    return X, np.r_[np.ones(n_per), -np.ones(n_per)]


def classifier_table():
    warnings.simplefilter('ignore')       # scikit-learn's deprecation notices
    try:
        from sklearn.linear_model import LogisticRegression
        from sklearn.preprocessing import StandardScaler
    except ImportError:
        LogisticRegression = None
    for n_per, d in [(500, 17), (1000, 50), (20000, 160)]:
        X, y = problem(n_per, d)
        Xd = torch.as_tensor(X, device='cuda')
        yd = torch.as_tensor(y, device='cuda')
        q = Xd[:1]
        out = torch.empty(ops.logreg_block_size(d) + 1, dtype=torch.float64, device='cuda')

        def run():
            f = ops.logreg_fit(Xd, yd, out=out[:-1])
            ops.logreg_predict(f, q, out=out[-1:])
            return f
        reps = 2 if d == 160 else 10
        med, lo, hi = device_ms(run, reps=reps)
        f = run()
        print('device fit+predict  rows/class {:6d} d {:3d}: {:9.3f} ms (min {:.3f}, max {:.3f}), '
              '{} Newton steps, converged {}'.format(n_per, d, med, lo, hi, f.n_iter, f.converged))
        if LogisticRegression is not None:
            ts = []
            for _ in range(3):
                t0 = time.perf_counter()
                Xs = StandardScaler().fit_transform(X)
                clf = LogisticRegression(penalty='l1', solver='liblinear').fit(Xs, y)
                clf.predict_proba(Xs[:1])
                ts.append(1e3 * (time.perf_counter() - t0))
            print('host liblinear      rows/class {:6d} d {:3d}: {:9.3f} ms (tol 1e-4, {} '
                  'iterations)'.format(n_per, d, float(np.median(ts)), int(clf.n_iter_[0])))


def round_split():
    m, _ = arch.get_device_model(n_obs=100, true_params=[0.3, 0.7], seed_obs=5)
    b = bf.BOLFIRE(m, 500, bounds={'t1': (-1, 1), 't2': (0, 1)}, n_initial_evidence=5, seed=3,
                   seed_marginal=4)
    b.fit(12, bar=False)          # warm-up: past the initial evidence, the acquisition runs
    parts = {'simulation': [], 'classifier': [], 'GP update + acquisition': []}
    for _ in range(8):            # one round, its pieces timed by hand
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        b._init_round()             # the LCBSC acquisition of the round's parameter
        t1 = time.perf_counter()
        batch = b._run_batch(b._next_batch_index, b.prepare_new_batch(b._next_batch_index))
        b._next_batch_index += 1
        b._merge_batch(batch)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        neg = -b._log_ratio()       # fit, predict and the round's one read
        t3 = time.perf_counter()
        b.classifier_attributes.append(b.classifier.attributes)
        b.state['n_evidence'] += 1
        b.target_model.update(b.current_params, neg, b._should_optimize())
        torch.cuda.synchronize()
        t4 = time.perf_counter()
        parts['simulation'].append(1e3 * (t2 - t1))
        parts['classifier'].append(1e3 * (t3 - t2))
        parts['GP update + acquisition'].append(1e3 * (t4 - t3 + t1 - t0))
    for k, v in parts.items():
        print('device ARCH round, 500 rows/class: {:24s} {:8.3f} ms (median of 8)'.format(
            k, float(np.median(v))))


if __name__ == '__main__':
    print('card:', card())
    classifier_table()
    round_split()
