"""Time the device regression adjustment (ops.linear_adjust) by stage with CUDA events: the row
mask, the moments, the host solve and the adjusted columns, at N in {1e5, 1e6, 1e7},
q in {2, 16, 128} and p in {2, 8}, every value finite (one group, dense output).  Each stage is
warmed up once and timed as the median of --repeats runs.  Bytes are the least each stage must
move (mask: S and theta once; moments: S and theta twice; adjust: S and theta once plus the
output), reported against the H100 SXM's 3.35 TB/s.  Prints the card's name and power limit, then
one JSON line per shape.  With ELFI_REFERENCE_ROOT set it also times the reference's host path
(its LinearAdjustment on the same arrays copied to the host) where N q <= 2e7.

    python scripts/time_adjust.py [--N 100000 1000000 10000000] [--q 2 16 128] [--p 2 8]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from elfi_b200 import _lib, ops  # noqa: E402
from elfi_b200 import device as dev  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else torch.cuda.get_device_name(0)


def timed(fn, repeats):
    fn()
    ms = []
    for _ in range(repeats):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        start.record()
        fn()
        end.record()
        torch.cuda.synchronize()
        ms.append(start.elapsed_time(end))
    return float(np.median(ms))


def run(N, q, p, repeats):
    g = torch.Generator(device='cuda').manual_seed(N + 7 * q + p)
    S = torch.randn((N, q), dtype=torch.float64, device='cuda', generator=g)
    T = S[:, :1].repeat(1, p) * 0.5 + torch.randn((N, p), dtype=torch.float64, device='cuda',
                                                  generator=g)
    o = torch.zeros(q, dtype=torch.float64, device='cuda')
    d = q + p
    ctx, stream = dev.context(), dev.stream_ptr()
    shape = (dev.ptr(S), q, N, q, dev.ptr(o), dev.ptr(T), p, p)
    flags = dev.empty((N,), dtype=torch.uint8)
    counts = dev.empty((p + 1,), dtype=torch.int64)
    cols = np.arange(p, dtype=np.int32)
    cptr = ctypes.c_void_p(cols.ctypes.data)
    mom = dev.empty((1 + d + d * d,))
    out = dev.empty((p, N))
    t = {}
    t['mask_ms'] = timed(lambda: _lib.call('elfi_b200_regadj_mask_f64', ctx, *shape,
                                           dev.ptr(flags), dev.ptr(counts), stream), repeats)
    t['moments_ms'] = timed(lambda: _lib.call('elfi_b200_regadj_moments_f64', ctx, *shape,
                                              dev.ptr(flags), cptr, p, -1, dev.ptr(mom), stream),
                            repeats)
    h = dev.to_host(mom)
    t0 = time.perf_counter()
    coef, _, _ = ops._regadj_solve(h[1 + d:].reshape(d, d), q, N, 1e-6)
    t['solve_host_ms'] = 1e3 * (time.perf_counter() - t0)
    coef_d = dev.to_device(np.ascontiguousarray(coef))
    t['adjust_ms'] = timed(lambda: _lib.call('elfi_b200_regadj_adjust_f64', ctx, *shape,
                                             dev.ptr(flags), cptr, p, -1, 1, dev.ptr(coef_d),
                                             dev.ptr(out), N, stream), repeats)
    t['linear_adjust_ms'] = timed(lambda: ops.linear_adjust(S, T, o), repeats)
    nbytes = {'mask': N * d * 8 + N, 'moments': 2 * N * d * 8 + 2 * N,
              'adjust': N * d * 8 + N + N * p * 8}
    rec = dict(N=N, q=q, p=p, **{k: round(v, 4) for k, v in t.items()})
    for k, b in nbytes.items():
        rec[k + '_bytes'] = b
        rec[k + '_share_of_hbm'] = round(b / HBM_BYTES_PER_S / (t[k + '_ms'] * 1e-3), 4)
    if os.environ.get('ELFI_REFERENCE_ROOT') and N * q <= 2e7:
        rec['reference_host_s'] = reference_time(S, T, o)
    del S, T, out
    torch.cuda.empty_cache()
    return rec


def reference_time(S, T, o):
    sys.path.insert(0, os.path.join(ROOT, 'oracle'))
    from ref_shim import import_reference
    import_reference()
    from elfi.methods import results
    from elfi.methods.post_processing import LinearAdjustment
    Sh, Th, oh = S.cpu().numpy(), T.cpu().numpy(), o.cpu().numpy()
    snames = ['s{}'.format(j) for j in range(Sh.shape[1])]
    pnames = ['t{}'.format(k) for k in range(Th.shape[1])]
    outputs = dict(zip(snames, Sh.T.copy()))
    outputs.update(zip(pnames, Th.T.copy()))
    sample = results.Sample(method_name='x', outputs=outputs, parameter_names=pnames)
    model = {s: types.SimpleNamespace(observed=np.array([v])) for s, v in zip(snames, oh)}
    t0 = time.perf_counter()
    adj = LinearAdjustment()
    adj.fit(sample, model, snames, pnames)
    adj.adjust()
    return round(time.perf_counter() - t0, 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--N', type=int, nargs='+', default=[10 ** 5, 10 ** 6, 10 ** 7])
    ap.add_argument('--q', type=int, nargs='+', default=[2, 16, 128])
    ap.add_argument('--p', type=int, nargs='+', default=[2, 8])
    ap.add_argument('--repeats', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('time_adjust.py needs a CUDA device')
    print(json.dumps({'card': card()}))
    for N in args.N:
        for q in args.q:
            for p in args.p:
                print(json.dumps(run(N, q, p, args.repeats)), flush=True)


if __name__ == '__main__':
    main()
