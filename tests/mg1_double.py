"""CPU test double of the M/G/1 and conditional-prior entry points -- TEST INFRASTRUCTURE ONLY.

Extends tests/abi_double.py and tests/priors_double.py (TABLE goes after theirs) with
restatements, on host pointers, of elfi_b200_sim_mg1_f64 and elfi_b200_row_quantiles_f64 (the
reference's recurrence and np.quantile; uniforms from a NumPy RandomState instead of the device's
Philox streams, same distribution, deterministic in (seed, offset)) and of
elfi_b200_prior_rvs_cond_f64, elfi_b200_prior_logpdf_cond_f64 and the mixture proposals with
support 4 (SciPy draws and densities with per-row loc / scale).
"""
import numpy as np
import scipy.stats as ss

import abi_double as d
import conditional_prior_replay as cr
import prior_replay as pr
import priors_double
from elfi_b200 import ops


def mg1_data(P, n, rs):
    """The reference's recurrence (mg1.py:37-54) on W, U drawn per row; NaN rows where it raises."""
    B = P.shape[0]
    u, v = 1.0 - rs.random_sample((B, n)), 1.0 - rs.random_sample((B, n))
    with np.errstate(all='ignore'):
        inv = 1 / P[:, 2]
        rng = P[:, 1] - P[:, 0]
        W = inv[:, None] * -np.log(u)
        U = P[:, 0, None] + rng[:, None] * v
        y = np.zeros((B, n))
        sw, sx = np.zeros(B), np.zeros(B)
        for j in range(n):
            sw += W[:, j]
            y[:, j] = U[:, j] + np.maximum(0, sw - sx)
            sx += y[:, j]
    bad = (np.signbit(inv) & ~np.isnan(inv)) | ~np.isfinite(rng)
    y[bad] = np.nan
    return y


def _q(q_host, nq):
    q = np.array(d._vec(q_host, nq))
    d._require(np.all((q >= 0) & (q <= 1)), 'every q must lie in [0, 1]')
    return q


def sim_mg1_f64(ctx, P, ldP, B, n_obs, nq, q_host, seed, offset, Y, ldY, S, ldS, stream):
    d._require(ldP >= 3 and ops.MG1_NOBS_MIN <= n_obs <= ops.MG1_NOBS_MAX, 'sim_mg1: bad shape')
    d._require(not d._addr(S) or (1 <= nq <= ops.MG1_NQ_MAX and ldS >= nq), 'sim_mg1: bad shape')
    q = _q(q_host, nq) if d._addr(S) else None
    if not B:
        return
    y = mg1_data(np.array(d._mat(P, B, 3, ldP)), n_obs, d._rs(seed, offset, 41))
    if d._addr(Y):
        d._mat(Y, B, n_obs, ldY)[:] = y
    if d._addr(S):
        d._mat(S, B, nq, ldS)[:] = np.quantile(y, q, axis=1).T


def row_quantiles_f64(ctx, X, ld_b, ld_j, B, n, nq, q_host, S, ldS, stream):
    d._require(ops.MG1_NOBS_MIN <= n <= ops.MG1_NOBS_MAX and 1 <= nq <= ops.MG1_NQ_MAX and ldS >= nq,
               'row_quantiles: bad shape')
    q = _q(q_host, nq)
    if not B:
        return
    span = (B - 1) * ld_b + (n - 1) * ld_j + 1
    x = np.array(np.lib.stride_tricks.as_strided(d._vec(X, span), (B, n), (8 * ld_b, 8 * ld_j)))
    d._mat(S, B, nq, ldS)[:] = np.quantile(x, q, axis=1).T


def _table7(spec_host, p):
    t = d._mat(spec_host, p, 7).copy()
    try:
        ops._prior_table(t[:, :5], t[:, 5:])
    except ValueError as e:
        d._require(False, str(e))
    return t


def prior_rvs_cond_f64(ctx, spec_host, B, seed, offset, loc, scale, out, stream):
    spec = d._mat(spec_host, 1, 5)[0].copy()
    why = ops._prior_spec_error(spec, 0 if d._addr(loc) else -1, 0 if d._addr(scale) else -1)
    d._require(why is None, 'prior parameter 0: {}'.format(why))
    if not B:
        return
    kind, shapes, l0, s0 = pr.unpack(spec)
    lv = np.array(d._vec(loc, B)) if d._addr(loc) else l0
    sv = np.array(d._vec(scale, B)) if d._addr(scale) else s0
    y = getattr(ss, kind).rvs(*shapes, size=B, random_state=d._rs(seed, offset, 7))
    with np.errstate(all='ignore'):
        x = lv + sv * y
    d._vec(out, B)[:] = np.where(sv >= 0, x, np.nan)


def prior_logpdf_cond_f64(ctx, x, ldx, B, p, spec_host, out, stream):
    t = _table7(spec_host, p)
    if B:
        d._vec(out, B)[:] = cr.joint_logpdf(t, d._mat(x, B, p, ldx))


def gm_rvs_cdf_f64(ctx, means, ldm, cumw, N, p, Lchol_host, B, seed, offset, support, box_host, out,
                   ldo, stream):
    if support != 4:
        return priors_double.gm_rvs_cdf_f64(ctx, means, ldm, cumw, N, p, Lchol_host, B, seed, offset,
                                            support, box_host, out, ldo, stream)
    c = d._vec(cumw, N)
    w = np.diff(np.concatenate([[0.0], c]))
    specs = _table7(box_host, p)
    rs = d._rs(seed, offset, 8)
    mu = d._mat(means, N, p, ldm)
    L = d._mat(Lchol_host, p, p)
    res = d._mat(out, B, p, ldo)
    todo = np.arange(B)
    for _ in range(1000):
        comp = rs.choice(N, size=len(todo), p=w / w.sum())
        draw = mu[comp] + rs.randn(len(todo), p) @ L.T
        ok = np.isfinite(cr.joint_logpdf(specs, draw))
        res[todo] = draw
        todo = todo[~ok]
        if not len(todo):
            break


TABLE = {'elfi_b200_' + f.__name__: f for f in (sim_mg1_f64, row_quantiles_f64, prior_rvs_cond_f64,
                                                 prior_logpdf_cond_f64, gm_rvs_cdf_f64)}
