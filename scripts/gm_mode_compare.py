#!/usr/bin/env python
"""Accuracy of the mixed-precision mixture density against the fp64 path (same inputs, two
processes: bench_out/gm_logq_<tag>.npy written by scripts/bench_r2_kernels.py)."""
import json
import sys

import numpy as np

a = np.load('bench_out/gm_logq_{}.npy'.format(sys.argv[1]))
b = np.load('bench_out/gm_logq_{}.npy'.format(sys.argv[2]))
rel = np.abs(np.expm1(b - a))
print(json.dumps({'name': 'gm_mode_accuracy', 'reference': sys.argv[1], 'variant': sys.argv[2],
                  'max_rel_err_density': float(rel.max()), 'median_rel_err_density': float(np.median(rel)),
                  'n': int(len(a))}))
