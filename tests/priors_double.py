"""CPU test double of the stock-prior entry points -- TEST INFRASTRUCTURE ONLY.

Extends tests/abi_double.py (through `abi_double.install`) with restatements of
elfi_b200_prior_rvs_f64, elfi_b200_prior_logpdf_f64 and the mixture proposals with support 3
(the prior table) on host pointers: scipy.stats draws and densities instead of the device's
Philox streams, so only statistical assertions apply.  Every other call goes to abi_double
unchanged (its gm_rvs is already generic in p for supports 0-2).
"""
import numpy as np
import scipy.stats as ss

import abi_double as d
import prior_replay as pr
from elfi_b200 import ops


def _table(spec_host, p):
    t = d._mat(spec_host, p, 5).copy()
    for i, row in enumerate(t):
        why = ops._prior_spec_error(row)
        d._require(why is None, 'prior parameter {}: {}'.format(i, why))
    return t


def prior_rvs_f64(ctx, spec_host, B, seed, offset, out, stream):
    spec = _table(spec_host, 1)[0]
    if not B:
        return
    kind, shapes, loc, scale = pr.unpack(spec)
    d._vec(out, B)[:] = getattr(ss, kind).rvs(*shapes, loc, scale, size=B,
                                              random_state=d._rs(seed, offset, 7))


def prior_logpdf_f64(ctx, x, ldx, B, p, spec_host, out, stream):
    t = _table(spec_host, p)
    if B:
        d._vec(out, B)[:] = pr.joint_logpdf(t, d._mat(x, B, p, ldx))


def gm_rvs_cdf_f64(ctx, means, ldm, cumw, N, p, Lchol_host, B, seed, offset, support, box_host, out,
                   ldo, stream):
    if support != 3:
        return d.gm_rvs_cdf_f64(ctx, means, ldm, cumw, N, p, Lchol_host, B, seed, offset, support,
                                box_host, out, ldo, stream)
    c = d._vec(cumw, N)
    w = np.diff(np.concatenate([[0.0], c]))
    specs = _table(box_host, p)
    rs = d._rs(seed, offset, 8)
    mu = d._mat(means, N, p, ldm)
    L = d._mat(Lchol_host, p, p)
    res = d._mat(out, B, p, ldo)
    todo = np.arange(B)
    for _ in range(1000):
        comp = rs.choice(N, size=len(todo), p=w / w.sum())
        draw = mu[comp] + rs.randn(len(todo), p) @ L.T
        ok = np.isfinite(pr.joint_logpdf(specs, draw))
        res[todo] = draw
        todo = todo[~ok]
        if not len(todo):
            break


TABLE = {'elfi_b200_prior_rvs_f64': prior_rvs_f64, 'elfi_b200_prior_logpdf_f64': prior_logpdf_f64,
         'elfi_b200_gm_rvs_cdf_f64': gm_rvs_cdf_f64}
