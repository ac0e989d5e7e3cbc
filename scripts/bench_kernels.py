#!/usr/bin/env python
"""Per-kernel device timings at the BASELINE shapes (CUDA events, warm, inputs > L2 or noted).
Writes bench_out/kernels.json.  Not the headline bench."""
import ctypes
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from elfi_b200 import _lib, ops  # noqa: E402
from elfi_b200 import device as dev  # noqa: E402

HBM = json.load(open(os.path.join(ROOT, 'MEASURED_PEAKS.json')))['hbm_gbs'] \
    if os.path.exists(os.path.join(ROOT, 'MEASURED_PEAKS.json')) else 6650.0


def timeit(fn, reps=7, warm=3, per_batch=10):
    """Median / min ms per call over `reps` batches of `per_batch` back-to-back calls between two
    CUDA events: the per-call Python and event overhead overlaps with the previous kernel instead
    of sitting inside the timing (round 1 timed single calls and read 0.19 ms where bench.py's
    device-timed loop measured 0.16 ms for the same kernel)."""
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(per_batch):
            fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) / per_batch)
    return float(np.median(ts)), float(np.min(ts))


def main():
    out = []
    gen = torch.Generator(device='cuda').manual_seed(0)
    peaks = (ctypes.c_double * 2)()
    _lib.call('elfi_b200_probe_fp64_f64', dev.context(), peaks)
    dfma, dmma = peaks[0], peaks[1]
    out.append(dict(name='fp64_peak_probe', dfma_tflops=dfma, dmma_tflops=dmma))

    def rec(name, ms, best, bytes_=None, flops=None, **kw):
        e = dict(name=name, ms_median=ms, ms_min=best, **kw)
        if bytes_ is not None:
            e['algorithmic_GB'] = bytes_ / 1e9
            e['GBps'] = bytes_ / (ms * 1e-3) / 1e9
            e['frac_hbm_measured'] = e['GBps'] / HBM
        if flops is not None:
            e['TFLOPs'] = flops / (ms * 1e-3) / 1e12
            e['frac_dfma_peak'] = e['TFLOPs'] / dfma
        out.append(e)
        print(json.dumps(e), flush=True)

    # K1: 1e6 x 128 euclid (+threshold mask)
    B, D = 1_000_000, 128
    S = torch.randn(B, D, dtype=torch.float64, device='cuda', generator=gen)
    obs = torch.randn(D, dtype=torch.float64, device='cuda', generator=gen)
    ms, best = timeit(lambda: ops.dist_euclid(S, obs))
    rec('K1 euclid 1e6x128', ms, best, bytes_=B * D * 8 + B * 8)
    # weighted K=1
    w = torch.rand(D, dtype=torch.float64, device='cuda', generator=gen) + 0.5
    ms, best = timeit(lambda: ops.dist_euclid(S, obs, w=w))
    rec('K4 weighted K=1 1e6x128', ms, best, bytes_=B * D * 8 + B * 8)
    del S
    # K4: nested K=5, 5e5 x 256 (config #5 per-GPU shard)
    B5, D5, K5 = 500_000, 256, 5
    S5 = torch.randn(B5, D5, dtype=torch.float64, device='cuda', generator=gen)
    obs5 = torch.randn(D5, dtype=torch.float64, device='cuda', generator=gen)
    W5 = torch.rand(K5, D5, dtype=torch.float64, device='cuda', generator=gen) + 0.5
    ms, best = timeit(lambda: ops.dist_euclid(S5, obs5, w=W5))
    rec('K4 nested K=5 5e5x256', ms, best, bytes_=B5 * D5 * 8 + B5 * K5 * 8,
        flops=B5 * D5 * (2 + 2 * K5))
    ms, best = timeit(lambda: ops.colmoments(S5))
    rec('K5 colmoments 5e5x256', ms, best, bytes_=B5 * D5 * 8)
    del S5
    # K6: autocov(1,2) 1e6 x 100 ; meanvar 1e6 x 50
    X = torch.randn(1_000_000, 100, dtype=torch.float64, device='cuda', generator=gen)
    ms, best = timeit(lambda: ops.autocov(X, lags=(1, 2)))
    rec('K6 autocov lags(1,2) 1e6x100', ms, best, bytes_=1_000_000 * 100 * 8 + 16_000_000)
    Y = torch.randn(1_000_000, 50, dtype=torch.float64, device='cuda', generator=gen)
    ms, best = timeit(lambda: ops.meanvar(Y))
    rec('K6 meanvar 1e6x50 (2 sweeps, 2nd from L2)', ms, best, bytes_=1_000_000 * 50 * 8 + 16_000_000)
    del X, Y
    # K3: argsort 2e6 keys ; K7 weighted quantile 1e6
    keys = torch.rand(2_000_000, dtype=torch.float64, device='cuda', generator=gen) * 20
    ms, best = timeit(lambda: ops.argsort(keys))
    rec('K3 argsort 2e6 fp64 keys', ms, best, keys_per_s=2e6 / (ms * 1e-3))
    k1 = keys[:1_000_000].contiguous()
    wts = torch.rand(1_000_000, dtype=torch.float64, device='cuda', generator=gen)
    ms, best = timeit(lambda: ops.weighted_sample_quantile(k1, 0.5, wts), reps=5)
    rec('K7 weighted quantile 1e6 (exact sequential cumsum)', ms, best)
    k10k = keys[:10_000].contiguous()
    ms, best = timeit(lambda: ops.argsort(k10k))
    rec('K3 argsort 1e4 keys (latency floor)', ms, best)
    # K8: weighted stats 1e6 x 2
    P = torch.randn(1_000_000, 2, dtype=torch.float64, device='cuda', generator=gen)
    ms, best = timeit(lambda: ops.weighted_stats(P, wts))
    rec('K8 weighted stats 1e6x2', ms, best)
    # K9: GM logpdf, N = M = 1e5 (1e10 pair terms); 16 fp64 ops per pair at p = 2
    N = M = 100_000
    x = torch.randn(N, 2, dtype=torch.float64, device='cuda', generator=gen)
    mns = torch.randn(M, 2, dtype=torch.float64, device='cuda', generator=gen)
    wm = torch.rand(M, dtype=torch.float64, device='cuda', generator=gen)
    cov = np.diag([0.05, 0.02])
    ms, best = timeit(lambda: ops.gm_logpdf(x, mns, cov, wm), reps=3, warm=1, per_batch=1)
    rec('K9 gm_logpdf N=M=1e5 p=2', ms, best, flops=N * M * 16 * 2.0,
        pair_terms_per_s=N * M / (ms * 1e-3),
        extrapolated_ms_N1e6_M1e6=ms * 100, note='fp64 ops/pair = 16 (flops = 2x for fma)')
    # K10-K12: GP fit n = 2000, predict 1e5 grid
    from elfi_b200.bo import GPyRegression
    rs = np.random.RandomState(0)
    Xe = rs.uniform([-2, -1], [2, 1], (2000, 2))
    ye = np.log(0.05 + np.sum((Xe - 0.3) ** 2, axis=1)) + 0.1 * rs.randn(2000)
    gp = GPyRegression(['t1', 't2'], bounds={'t1': (-2, 2), 't2': (-1, 1)})
    gp.update(Xe, ye)
    ms, best = timeit(lambda: gp._fit(), reps=5, warm=2, per_batch=3)
    n = 2000
    rec('K10+K11 GP fit n=2000 (gram+chol+inverse+alpha)', ms, best,
        flops=(n ** 3 / 3 + 2 * n ** 3 / 3) * 2.0 / 2 * 2, note='~n^3/3 chol + ~2n^3/3 inverse FMAs')
    g1, g2 = np.meshgrid(np.linspace(-2, 2, 400), np.linspace(-1, 1, 250))
    grid = dev.to_device(np.column_stack([g1.ravel(), g2.ravel()]))
    ms, best = timeit(lambda: gp.predict_device(grid, noiseless=True, beta=20.0), reps=5, warm=2, per_batch=3)
    m = grid.shape[0]
    rec('K12 GP predict + LCBSC m=1e5 n=2000', ms, best, flops=(m * n * n / 2 + m * n) * 2.0,
        frac_dmma_peak=(m * n * n / 2 + m * n) * 2.0 / (ms * 1e-3) / 1e12 / dmma)
    xq = grid[:10].contiguous()
    ms, best = timeit(lambda: gp.predict_device(xq, noiseless=True, beta=20.0), reps=5, warm=2, per_batch=3)
    rec('GP predict + LCBSC m=10 n=2000 (row-parallel path)', ms, best)
    xq128 = grid[:128].contiguous()
    ms, best = timeit(lambda: gp.predict_device(xq128, noiseless=True, beta=20.0), reps=5, warm=2, per_batch=3)
    rec('GP predict + LCBSC m=128 n=2000 (GEMM path)', ms, best)
    ms, best = timeit(lambda: gp._predict_grad_device(xq), reps=5, warm=2, per_batch=3)
    rec('K13 GP predictive gradients m=10 n=2000', ms, best)
    try:
        # ---- kernels added after round 1's last GPU session (first timings in round 2)
        from elfi_b200.bo import LCBSC
        acq = LCBSC(gp, seed=0)
        ms, best = timeit(lambda: acq.evaluate_with_gradient(xq.cpu().numpy(), 5), reps=5, warm=2, per_batch=3)
        rec('LCBSC value+gradient m=10 n=2000 (one lock-step acquisition round, incl. D2H)', ms, best)
        pts = grid[:200].contiguous()
        ms, best = timeit(lambda: gp.whiten(pts), reps=5, warm=2, per_batch=3)
        rec('gp_whiten m=200 n=2000', ms, best, flops=200 * n * n)
        wh = gp.whiten(pts)
        one = gp.whiten(grid[777:778].contiguous())
        ms, best = timeit(lambda: gp.cross_covariance(wh, one), reps=5, warm=2, per_batch=3)
        rec('gp_cross_cov 200 x 1, n=2000', ms, best)
        count = [0]

        def append_one():      # n = 2000 -> 2007: stays inside the padded size 2048
            xn = np.array([[0.31 + 0.01 * count[0], 0.17]])
            count[0] += 1
            gp._X, gp._Y = np.r_[gp._X, xn], np.r_[gp._Y, np.array([[0.2]])]
            if not gp._append(xn, np.array([[0.2]])):
                raise RuntimeError('rank-1 update refused')
        ms, best = timeit(append_one, reps=5, warm=2, per_batch=3)
        rec('GP rank-1 factor update n~2000 (vs the refit above)', ms, best)
        S = torch.randn(B, D, dtype=torch.float64, device='cuda', generator=gen)
        for metric, pexp in (('sqeuclidean', 2.0), ('cityblock', 2.0), ('chebyshev', 2.0),
                             ('minkowski', 3.0)):
            ms, best = timeit(lambda: ops.dist_metric(S, obs, metric, p=pexp))
            rec('dist_metric {} 1e6x128'.format(metric), ms, best, bytes_=B * D * 8 + B * 8)
        del S
        par = [torch.rand(1_000_000, dtype=torch.float64, device='cuda', generator=gen) * 10
               for _ in range(4)]
        ms, best = timeit(lambda: ops.sim_gnk(*par, n_obs=256, seed=1), reps=5, warm=2, per_batch=3)
        rec('sim_gnk 1e6 x 256 (write only)', ms, best, bytes_=1_000_000 * 256 * 8)
        Y = ops.sim_gnk(*par, n_obs=256, seed=1)
        ms, best = timeit(lambda: ops.rowsort(Y), reps=5, warm=2, per_batch=3)
        rec('rowsort 1e6 x 256', ms, best, bytes_=2 * 1_000_000 * 256 * 8)
        del Y, par
        xs = torch.rand(1_000_000, dtype=torch.float64, device='cuda', generator=gen)
        ms, best = timeit(lambda: ops.weighted_sample_quantile(xs, 0.5))
        rec('weighted quantile 1e6, equal weights (closed-form position)', ms, best)
    except Exception as exc:   # keep the timings gathered so far
        out.append(dict(name='new-kernel section failed', error=repr(exc)))
        print(json.dumps(out[-1]), flush=True)
    os.makedirs(os.path.join(ROOT, 'bench_out'), exist_ok=True)
    with open(os.path.join(ROOT, 'bench_out', 'kernels.json'), 'w') as f:
        json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
