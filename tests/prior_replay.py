"""NumPy replay of the stock-prior streams (elfi_b200/csrc/prior.cu) and of the mixture proposals
for p <= 16 and support 3 (gm_rvs_wide_kernel in simulate.cu) -- TEST INFRASTRUCTURE ONLY.

Built on oracle/streams.py (the Philox generator, u01 and Box-Muller, which are pinned there);
it follows each kernel's counter layout word for word so that tests/test_device_priors_gpu.py can
compare the device draws with it element by element.  The inverse normal CDF is
scipy.special.ndtri, the log densities are scipy.stats'.
"""
import numpy as np
import scipy.stats as ss
from scipy.special import erfc, ndtri

import streams

SALT_PRIOR = 0x50524F52
SALT_GM_RVS_WIDE = 0x474D5258
KINDS = ('uniform', 'norm', 'truncnorm', 'expon', 'gamma', 'beta')
NSHAPE = {'uniform': 0, 'norm': 0, 'truncnorm': 2, 'expon': 0, 'gamma': 1, 'beta': 2}
MAX_TRIALS = 64
EPS = 2.0 ** -52


def unpack(spec):
    """(kind name, shapes, loc, scale) of a [kind, p0, p1, p2, p3] row."""
    kind = KINDS[int(spec[0])]
    ns = NSHAPE[kind]
    return kind, tuple(float(v) for v in spec[1:1 + ns]), float(spec[1 + ns]), float(spec[2 + ns])


def scipy_logpdf(spec, x):
    kind, shapes, loc, scale = unpack(spec)
    with np.errstate(all='ignore'):
        return getattr(ss, kind).logpdf(x, *shapes, loc, scale)


def joint_logpdf(specs, x):
    """Sum, left to right, of the per-column scipy log densities."""
    out = None
    for a, spec in enumerate(specs):
        t = scipy_logpdf(spec, x[:, a])
        out = t if out is None else out + t
    return out


def support(spec):
    """Closed support [lo, hi] of a parameter in x units."""
    kind, shapes, loc, scale = unpack(spec)
    lo, hi = {'uniform': (0.0, 1.0), 'norm': (-np.inf, np.inf), 'expon': (0.0, np.inf),
              'gamma': (0.0, np.inf), 'beta': (0.0, 1.0)}.get(kind, shapes)
    return loc + lo * scale, loc + hi * scale


def gamma_constants(s):
    """Marsaglia-Tsang (d, c, inv_a) of G(s): s < 1 is drawn as G(s + 1) u^(1/s)."""
    inv_a = 1.0 / s if s < 1.0 else 0.0
    d = (s + 1.0 if s < 1.0 else s) - 1.0 / 3.0
    return d, 1.0 / np.sqrt(9.0 * d), inv_a


def mt_trial(d, c, z, u):
    """One Marsaglia-Tsang trial per element (priors.cuh's prior_mt_accept):
    (accepted, v, margin |bound - log u|, +inf where 1 + c z <= 0)."""
    t = 1.0 + c * z
    ok = t > 0.0
    with np.errstate(all='ignore'):
        v = t * t * t
        bound = 0.5 * z * z + d - d * v + d * np.log(v)
        lu = np.log(u)
    acc = ok & (lu < bound)
    margin = np.where(ok, np.abs(bound - lu), np.inf)
    return acc, np.where(ok, v, 0.0), margin


def gamma_component(rows, g, s, seed, max_trials=MAX_TRIALS):
    """G(s) of component g per row: trial t uses z = first normal of block (g << 16) | 2t and
    u = u01(x, y), w = u01(z, w) of block (g << 16) | (2t + 1).  Returns (G, trial (-1 when all
    trials were rejected), margin = the smallest acceptance margin up to the deciding trial,
    rel_err = a bound of the replay's relative error)."""
    d, c, inv_a = gamma_constants(s)
    n = rows.size
    v = np.ones(n)
    w = np.ones(n)
    zr = np.zeros(n)
    rad = np.zeros(n)
    trial = np.full(n, -1, dtype=np.int64)
    margin = np.full(n, np.inf)
    act = np.arange(n)
    for t in range(max_trials):
        if act.size == 0:
            break
        blk = (g << 16) | (2 * t)
        z, _, r = streams.normal2(streams._block(rows[act], blk, SALT_PRIOR, seed))
        q = streams._block(rows[act], blk + 1, SALT_PRIOR, seed)
        u, ww = streams.u01(q[0], q[1]), streams.u01(q[2], q[3])
        acc, vt, mg = mt_trial(d, c, z, u)
        margin[act] = np.minimum(margin[act], mg)
        hit = act[acc]
        v[hit], w[hit], zr[hit], rad[hit], trial[hit] = vt[acc], ww[acc], z[acc], r[acc], t
        act = act[~acc]
    G = d * v
    if inv_a > 0.0:
        G = G * np.power(w, inv_a)
    # z is within 1e-14 max(1, rad) of the device's: v = (1 + c z)^3 moves by 3 c dz / (1 + c z)
    tz = np.maximum(1.0 + c * zr, 1e-300)
    rel_err = 3.0 * c * 1e-14 * np.maximum(1.0, rad) / tz + 16 * EPS
    return G, trial, margin, rel_err


def prior_rvs(spec, B, seed, offset=0):
    """prior_rvs_kernel.  Returns (x (B,), err (B,) a bound of the replay's error, trial (B,) the
    deciding trial of the gamma components (the larger for beta; 0 for the other kinds), margin
    (B,) the smallest acceptance margin of the gamma trials (+inf for the other kinds))."""
    kind, shapes, loc, scale = unpack(spec)
    rows = streams.rows_of(B, offset)
    trial = np.zeros(B, dtype=np.int64)
    margin = np.full(B, np.inf)
    if kind in ('gamma', 'beta'):
        gx, tx, mx, ex = gamma_component(rows, 0, shapes[0], seed)
        if kind == 'gamma':
            y, trial, margin, rel = gx, tx, mx, ex
        else:
            gy, ty, my, ey = gamma_component(rows, 1, shapes[1], seed)
            y = gx / (gx + gy)
            trial, margin = np.maximum(tx, ty), np.minimum(mx, my)
            rel = 2 * (ex + ey) + 4 * EPS
        yerr = rel * np.abs(y)
    else:
        w = streams._block(rows, 0, SALT_PRIOR, seed)
        u = streams.u01(w[0], w[1])
        if kind == 'uniform':
            y, yerr = u, np.zeros(B)
        elif kind == 'norm':
            y, _, rad = streams.normal2(w)
            yerr = 1e-14 * np.maximum(1.0, rad)
        elif kind == 'truncnorm':
            a, b = shapes
            mirror = a > 0
            lo, hi = (-b, -a) if mirror else (a, b)
            r2 = 0.7071067811865476
            cdf_lo = 0.5 * erfc(-lo * r2)
            cdf_w = 0.5 * erfc(-hi * r2) - cdf_lo
            q = cdf_lo + u * cdf_w
            y = (-1.0 if mirror else 1.0) * np.minimum(np.maximum(ndtri(q), lo), hi)
            # both inverse CDFs are accurate to ~1e-14 relative, and the argument may differ by
            # an ulp or two (the device fuses u * cdf_w + cdf_lo): dy = dq / phi(y)
            yerr = 1e-13 * np.abs(y) + 4 * EPS * q / ss.norm.pdf(y)
        else:
            y = -np.log(u)
            yerr = 4 * EPS * np.abs(y) + 2 * EPS
    x = loc + scale * y
    err = scale * yerr + 4 * EPS * (abs(loc) + np.abs(scale * y))
    return x, err, trial, margin


def support_margin(specs, x):
    """(inside: the joint log density is finite, distance of the nearest coordinate to an edge of
    its support) of draws x (rows, p)."""
    inside = np.isfinite(joint_logpdf(specs, x))
    margin = np.full(x.shape[0], np.inf)
    for a, spec in enumerate(specs):
        lo, hi = support(spec)
        for edge in (lo, hi):
            if np.isfinite(edge):
                margin = np.minimum(margin, np.abs(x[:, a] - edge))
    return inside, margin


def gm_rvs(means, L, cumw, B, seed, offset=0, support_code=0, box=None, specs=None,
           max_trials=1000):
    """gm_rvs_wide_kernel (equal to gm_rvs_kernel for p <= 4 and supports 0-2).  Trial t: blocks
    4t, 4t + 1, 4t + 2 of SALT_GM_RVS as oracle/streams.gm_rvs; z_{4+2k}, z_{5+2k} from block
    8t + k of SALT_GM_RVS_WIDE.  Support 3 keeps draws whose joint prior log density is finite.
    Returns (x, trial, comp, err, margin) as streams.gm_rvs."""
    means = np.asarray(means, dtype=np.float64)
    L = np.asarray(L, dtype=np.float64)
    cumw = np.asarray(cumw, dtype=np.float64)
    p = means.shape[1]
    total = cumw[-1]
    rows = streams.rows_of(B, offset)
    x = np.zeros((B, p))
    err = np.zeros(B)
    comp = np.zeros(B, dtype=np.int64)
    trial = np.full(B, -1, dtype=np.int64)
    margin = np.full(B, np.inf)
    act = np.arange(B)
    npair = (p + 1) // 2
    for t in range(max_trials):
        if act.size == 0:
            break
        r = rows[act]
        w = streams._block(r, 4 * t, streams.SALT_GM_RVS, seed)
        c = streams._first_ge(cumw, streams.u01(w[0], w[1]) * total)
        z = np.zeros((act.size, 2 * npair + 2))
        rad = np.zeros((act.size, npair + 1))
        z[:, 0], z[:, 1], rad[:, 0] = streams.normal2(streams._block(r, 4 * t + 1, streams.SALT_GM_RVS, seed))
        if p > 2:
            z[:, 2], z[:, 3], rad[:, 1] = streams.normal2(streams._block(r, 4 * t + 2, streams.SALT_GM_RVS, seed))
        for k in range(max(0, npair - 2)):
            z[:, 4 + 2 * k], z[:, 5 + 2 * k], rad[:, 2 + k] = streams.normal2(
                streams._block(r, 8 * t + k, SALT_GM_RVS_WIDE, seed))
        zerr = 1e-14 * np.maximum(1.0, rad)[:, np.arange(2 * npair + 2) // 2]
        xt = np.empty((act.size, p))
        et = np.zeros(act.size)
        for a in range(p):
            s = means[c, a].copy()
            mag = np.abs(s)
            e = np.zeros(act.size)
            for b in range(a + 1):
                s = s + L[a, b] * z[:, b]
                mag = mag + np.abs(L[a, b] * z[:, b])
                e = e + abs(L[a, b]) * zerr[:, b]
            xt[:, a] = s
            et = np.maximum(et, e + 4 * EPS * mag)
        if support_code == 3:
            inside, mg = support_margin(specs, xt)
        else:
            inside, mg = streams._support_margin(xt, support_code, box)
        x[act], err[act], comp[act] = xt, et, c
        margin[act] = np.minimum(margin[act], mg)
        trial[act[inside]] = t
        act = act[~inside]
    return x, trial, comp, err, margin
