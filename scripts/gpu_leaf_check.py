"""One short GPU call: summary-kernel parity tests, then CUDA-event timings of the two
row-stream summary kernels on the benchmark shapes.  Writes bench_out/leaf_check.json."""
import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.makedirs(os.path.join(ROOT, 'bench_out'), exist_ok=True)
rc = pytest.main(['-x', '-q', '-m', 'gpu', os.path.join(ROOT, 'tests', 'test_summaries_gpu.py'),
                  os.path.join(ROOT, 'tests', 'test_model_gpu.py')])
res = {'pytest_rc': int(rc)}

import torch  # noqa: E402
from elfi_b200 import ops  # noqa: E402


def timed(fn, reps=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
    ev[0].record()
    for i in range(reps):
        fn()
        ev[i + 1].record()
    torch.cuda.synchronize()
    ts = sorted(ev[i].elapsed_time(ev[i + 1]) for i in range(reps))
    return ts[len(ts) // 2]


x = torch.randn(1_000_000, 100, dtype=torch.float64, device='cuda')
ms = timed(lambda: ops.autocov(x, lags=(1, 2)))
res['autocov_1e6x100_ms'] = ms
res['autocov_GBps'] = x.numel() * 8 / ms / 1e6
y = torch.randn(2_000_000, 50, dtype=torch.float64, device='cuda')
ms = timed(lambda: ops.meanvar(y))
res['meanvar_2e6x50_ms'] = ms
res['meanvar_GBps'] = y.numel() * 8 / ms / 1e6
z = torch.randn(400_000, 256, dtype=torch.float64, device='cuda')
ms = timed(lambda: ops.autocov(z, lags=(1, 2)))
res['autocov_tree_4e5x256_ms'] = ms
res['autocov_tree_GBps'] = z.numel() * 8 / ms / 1e6
print(json.dumps(res))
with open(os.path.join(ROOT, 'bench_out', 'leaf_check.json'), 'w') as f:
    json.dump(res, f, indent=1)
sys.exit(int(rc))
