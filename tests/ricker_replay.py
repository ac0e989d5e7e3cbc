"""NumPy replay of the Poisson sampler (elfi_b200/csrc/poisson.cuh) and of the Ricker streams
(elfi_b200/csrc/ricker.cu) -- TEST INFRASTRUCTURE ONLY.

Built on oracle/streams.py (the Philox generator, u01 and Box-Muller); it follows the kernels'
counter layouts and the sampler's order of operations word for word, vectorised over elements, so
that tests can compare the host build of poisson.cuh and the device with it element by element.
NumPy's exp / log may differ from the device's (and glibc's) in the last bit, so every decision
carries its margin; a draw whose smallest margin is below POISSON_MARGIN is ambiguous and is
excluded from exact comparisons (and counted).
"""
import numpy as np

import streams

SALT_POISSON = 0x504F4953
SALT_RICKER = 0x5249434B
LAM_MAX = 9.223372006484771e18
SWITCH = 10.0
INV_MAX = 64
MAX_TRIALS = 32
HALF_LOG_2PI = 0.9189385332046728
EPS = 2.0 ** -52
# decision margins below these may flip between two correct implementations of exp / log: the
# inversion compares u with a CDF that carries exp(-lam)'s relative error (a few ulp); the PTRS
# test compares two log values of magnitude <= ~50 whose errors are a few 1e-14
POISSON_MARGIN = {'inversion': 1e-12, 'ptrs': 1e-10}

_STIRLERR = np.array([np.nan, 0.08106146679532726, 0.0413406959554093, 0.02767792568499834,
                      0.020790672103765093, 0.016644691189821193, 0.013876128823070748,
                      0.01189670994589177, 0.010411265261972096, 0.009255462182712733,
                      0.00833056343336287, 0.007573675487951841, 0.00694284010720953,
                      0.006408994188004207, 0.0059513701127588475, 0.005554733551962801])


def stirlerr(n):
    n = np.asarray(n, dtype=np.float64)
    S0, S1, S2, S3, S4 = 1.0 / 12, 1.0 / 360, 1.0 / 1260, 1.0 / 1680, 1.0 / 1188
    with np.errstate(all='ignore'):
        nn = n * n
        big = (S0 - (S1 - (S2 - (S3 - S4 / nn) / nn) / nn) / nn) / n
    small = _STIRLERR[np.clip(n, 0, 15).astype(np.int64)]
    return np.where(n <= 15.0, small, big)


def bd0(x, m):
    x, m = np.broadcast_arrays(np.asarray(x, dtype=np.float64), np.asarray(m, dtype=np.float64))
    with np.errstate(all='ignore'):
        dx = x - m
        series = np.abs(dx) < 0.1 * (x + m)
        v = dx / (x + m)
        s = dx * v
        ej = 2.0 * x * v
        v = v * v
        live = series.copy()
        for j in range(1, 32):
            ej = ej * v
            s1 = s + ej / float(2 * j + 1)
            live &= s1 != s
            s = np.where(live, s1, s)
        direct = x * np.log(x / m) + (m - x)
    return np.where(series, s, direct)


def logpmf(k, lam):
    """log p(k; lam), Loader's form as poisson.cuh evaluates it."""
    k, lam = np.broadcast_arrays(np.asarray(k, dtype=np.float64), np.asarray(lam, dtype=np.float64))
    with np.errstate(all='ignore'):
        v = -(stirlerr(k) + bd0(k, lam)) - (HALF_LOG_2PI + 0.5 * np.log(k))
    return np.where(k == 0.0, -lam, v)


def logpmf_numpy_form(k, lam):
    """NumPy's PTRS acceptance bound -lam + k log(lam) - lgamma(k + 1) (random_poisson_ptrs)."""
    from scipy.special import gammaln
    return -lam + k * np.log(lam) - gammaln(k + 1)


def draw(lam, rows, seed, base, salt):
    """poisson_draw for rate lam[i] from the blocks (rows[i], base + j, salt): (k, trials, margin,
    kind) with kind 0 for the exact results (0 and NaN), 1 inversion, 2 PTRS."""
    lam = np.asarray(lam, dtype=np.float64).reshape(-1)
    rows = np.asarray(rows, dtype=np.uint64).reshape(-1)
    n = lam.size
    base = np.broadcast_to(np.asarray(base, dtype=np.uint64), (n,))
    k = np.zeros(n)
    trials = np.zeros(n, dtype=np.int64)
    margin = np.full(n, np.inf)
    kind = np.zeros(n, dtype=np.int64)
    bad = ~(lam >= 0.0) | (lam > LAM_MAX)
    k[bad] = np.nan
    inv = np.flatnonzero(~bad & (lam > 0.0) & (lam < SWITCH))
    if inv.size:
        kind[inv] = 1
        w = streams._block(rows[inv], base[inv], salt, seed)
        u = streams.u01(w[0], w[1])
        lm = lam[inv]
        p = np.exp(-lm)
        F = p.copy()
        kk = np.zeros(inv.size)
        mg = np.full(inv.size, np.inf)
        live = np.ones(inv.size, dtype=bool)
        for j in range(INV_MAX):
            mg = np.where(live, np.minimum(mg, np.abs(u - F) / F), mg)
            live &= ~(u <= F)
            if not live.any():
                break
            p = np.where(live, p * lm / float(j + 1), p)
            F = np.where(live, F + p, F)
            kk = np.where(live, j + 1.0, kk)
        k[inv], trials[inv], margin[inv] = kk, 1, mg
    pt = np.flatnonzero(~bad & (lam >= SWITCH))
    if pt.size:
        kind[pt] = 2
        lm = lam[pt]
        b = 0.931 + 2.53 * np.sqrt(lm)
        a = -0.059 + 0.02483 * b
        log_invalpha = np.log(1.1239 + 1.1328 / (b - 3.4))
        vr = 0.9277 - 3.6224 / (b - 2.0)
        kk = np.floor(lm)
        tr = np.full(pt.size, MAX_TRIALS)
        mg = np.full(pt.size, np.inf)
        act = np.arange(pt.size)
        for j in range(MAX_TRIALS):
            if act.size == 0:
                break
            w = streams._block(rows[pt[act]], base[pt[act]] + np.uint64(j), salt, seed)
            U = streams.u01(w[0], w[1]) - 0.5
            V = streams.u01(w[2], w[3])
            with np.errstate(all='ignore'):
                us = 0.5 - np.abs(U)
                kf = np.floor((2.0 * a[act] / us + b[act]) * U + lm[act] + 0.43)
                quick = (us >= 0.07) & (V <= vr[act])
                skip = ~quick & ((kf < 0.0) | ((us < 0.013) & (V > us)))
                test = ~quick & ~skip
                lhs = (np.log(V) + log_invalpha[act]) - np.log(a[act] / (us * us) + b[act])
                rhs = logpmf(np.where(test, kf, 1.0), lm[act])
            acc = quick | (test & (lhs <= rhs))
            mg[act] = np.where(test, np.minimum(mg[act], np.abs(lhs - rhs)), mg[act])
            kk[act[acc]] = kf[acc]
            tr[act[acc]] = j + 1
            act = act[~acc]
        k[pt], trials[pt], margin[pt] = kk, tr, mg
    return k, trials, margin, kind


def ambiguous(margin, kind):
    """Draws whose decisions are too close to call between two correct log / exp."""
    return ((kind == 1) & (margin < POISSON_MARGIN['inversion'])) | \
        ((kind == 2) & (margin < POISSON_MARGIN['ptrs']))


def poisson_ops(lam, seed, offset=0):
    """ops.poisson: element i uses row offset + i, blocks j = 0, 1, .. of SALT_POISSON."""
    lam = np.asarray(lam, dtype=np.float64).reshape(-1)
    return draw(lam, streams.rows_of(lam.size, offset), seed, 0, SALT_POISSON)


def ricker_normals(B, n_obs, seed, offset=0):
    """e_t of every row and step of the stochastic simulator (block t << 8), with the Box-Muller
    radius that bounds the replay's error (1e-14 max(1, rad))."""
    rows = streams.rows_of(B, offset)[:, None]
    t = (np.arange(n_obs, dtype=np.uint64) << np.uint64(8))[None, :]
    e, _, rad = streams.normal2(streams._block(rows, t, SALT_RICKER, seed))
    return e, rad


def ricker_counts(lam, B, n_obs, seed, offset=0):
    """The Poisson draw of every (row, step) at the given rates lam (B, n_obs): blocks
    (t << 8) | (1 + j) of SALT_RICKER.  Returns draw()'s tuple reshaped to (B, n_obs)."""
    rows = np.repeat(streams.rows_of(B, offset), n_obs)
    base = np.tile((np.arange(n_obs, dtype=np.uint64) << np.uint64(8)) | np.uint64(1), B)
    return tuple(v.reshape(B, n_obs) for v in draw(np.asarray(lam).reshape(-1), rows, seed, base,
                                                   SALT_RICKER))
