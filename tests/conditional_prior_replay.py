"""NumPy replay of the conditional priors (a loc or scale taken from another column of the row;
elfi_b200/csrc/priors.cuh) -- TEST INFRASTRUCTURE ONLY.

Extends tests/prior_replay.py: the per-row SciPy log densities of a (p, 7) table [kind, p0, p1, p2,
p3, loc_src, scale_src], the support margins of its proposals, the proposal replay of gm_rvs
support 4, and the exact fma of the per-row draw loc + scale y.
"""
from fractions import Fraction

import numpy as np
import scipy.stats as ss

import prior_replay as pr


def unpack(spec7, x):
    """(kind, shapes, loc, scale) of a 7-word row, loc and scale per row of x (n, p) where
    sourced."""
    kind, shapes, loc, scale = pr.unpack(spec7[:5])
    ls, ss_ = int(spec7[5]), int(spec7[6])
    if ls >= 0:
        loc = x[:, ls]
    if ss_ >= 0:
        scale = x[:, ss_]
    return kind, shapes, loc, scale


def scipy_logpdf(spec7, x, a):
    kind, shapes, loc, scale = unpack(spec7, x)
    with np.errstate(all='ignore'):
        return getattr(ss, kind).logpdf(x[:, a], *shapes, loc, scale)


def joint_logpdf(specs7, x):
    """Sum, left to right, of the per-column SciPy log densities with per-row loc / scale."""
    x = np.asarray(x, dtype=np.float64)
    out = None
    for a, spec in enumerate(specs7):
        t = scipy_logpdf(spec, x, a)
        out = t if out is None else out + t
    return out


def support_margin(specs7, x):
    """(inside: finite joint density, distance of the nearest coordinate to an edge of its
    per-row support) of draws x (rows, p)."""
    inside = np.isfinite(joint_logpdf(specs7, x))
    margin = np.full(x.shape[0], np.inf)
    for a, spec in enumerate(specs7):
        kind, shapes, loc, scale = unpack(spec, x)
        lo, hi = {'uniform': (0.0, 1.0), 'norm': (-np.inf, np.inf), 'expon': (0.0, np.inf),
                  'gamma': (0.0, np.inf), 'beta': (0.0, 1.0)}.get(kind, shapes)
        with np.errstate(all='ignore'):
            for edge in (lo, hi):
                if np.isfinite(edge):
                    margin = np.minimum(margin, np.abs(x[:, a] - (loc + edge * scale)))
    return inside, margin


def gm_rvs(means, L, cumw, B, seed, offset, specs7, max_trials=1000):
    """gm_rvs support 4: prior_replay.gm_rvs (the blocks of support 3) with the acceptance and
    margins of the per-row supports.  Returns (x, trial, comp, err, margin)."""
    saved = pr.support_margin
    pr.support_margin = lambda specs, x: support_margin(specs7, x)
    try:
        return pr.gm_rvs(means, L, cumw, B, seed, offset, 3, specs=specs7, max_trials=max_trials)
    finally:
        pr.support_margin = saved


def fma(a, b, c):
    """a * b + c rounded once, elementwise (exact rational arithmetic); NaN / inf as IEEE."""
    a, b, c = np.broadcast_arrays(*(np.asarray(v, dtype=np.float64) for v in (a, b, c)))
    out = np.empty(a.shape)
    with np.errstate(all='ignore'):
        naive = a * b + c
    for i in np.ndindex(a.shape):
        if np.isfinite(naive[i]) and np.isfinite(a[i] * b[i]):
            r = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
            out[i] = float(r) if r != 0 else naive[i]
        else:
            out[i] = naive[i]
    return out
