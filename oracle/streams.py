"""NumPy replay of the throughput-mode random streams (elfi_b200/csrc/simulate.cu).

TEST INFRASTRUCTURE ONLY -- ``elfi_b200`` never imports this module.

Every device prior, simulator and proposal draw is a pure function of (seed, row, block, salt):
one Philox4x32-10 block per counter (row, row >> 32, block, salt) keyed by the seed.  The
functions below follow each kernel's counter layout word for word, vectorised over rows, so that
tests/test_streams_gpu.py can compare the kernels with them element by element.  The generator and
the uniform conversion are exact (bit-identical to the device); Box-Muller uses an exactly reduced
sinpi / cospi so the replayed normals are within about one ulp of the correctly rounded value, and
everything downstream follows the kernel's order of operations.  A stream-layout mistake in a kernel
(a wrong counter word, a shared block, a wrong bit mapping) shows up as an O(1) difference.
"""
import numpy as np

_MASK32 = np.uint64(0xFFFFFFFF)
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)

SALT_PRIOR_MA2 = 0x50524931
SALT_SIM_MA2 = 0x4D413257
SALT_GM_RVS = 0x474D5256
SALT_PRIOR_GAUSS = 0x47415553
SALT_SIM_GAUSS = 0x47534D55
SALT_SIM_GNK = 0x474E4B30


def _u64(x):
    return np.asarray(x, dtype=np.uint64)


def philox4x32_10(c0, c1, c2, c3, seed):
    """Philox4x32-10 of counter (c0, c1, c2, c3), key (seed & 0xffffffff, seed >> 32); arguments
    broadcast.  Returns the four output words as uint64 arrays holding 32-bit values."""
    c0, c1, c2, c3, seed = np.broadcast_arrays(_u64(c0), _u64(c1), _u64(c2), _u64(c3), _u64(seed))
    c0, c1, c2, c3 = (c & _MASK32 for c in (c0, c1, c2, c3))
    k0, k1 = seed & _MASK32, seed >> np.uint64(32)
    for _ in range(10):
        p0 = _M0 * c0          # < 2^64: exact in uint64
        p1 = _M1 * c2
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _MASK32,
                          (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _MASK32)
        k0 = (k0 + _W0) & _MASK32
        k1 = (k1 + _W1) & _MASK32
    return c0, c1, c2, c3


def u01(a, b):
    """((a << 21) ^ (b >> 11)) + 1, times 2^-53: a uniform on (0, 1]; exact."""
    v = ((_u64(a) << np.uint64(21)) ^ (_u64(b) >> np.uint64(11))) & np.uint64((1 << 53) - 1)
    return (v.astype(np.float64) + 1.0) * 2.0 ** -53


def sincospi(x):
    """(sin(pi x), cos(pi x)) with the argument reduced exactly: x = n/2 + r, |r| <= 1/4."""
    x = np.asarray(x, dtype=np.float64)
    n = np.rint(2.0 * x)
    r = x - 0.5 * n                      # exact (x is a multiple of 2^-52 here, |r| <= 1/4)
    s, c = np.sin(np.pi * r), np.cos(np.pi * r)
    q = n.astype(np.int64) & 3
    sin = np.choose(q, [s, c, -s, -c])
    cos = np.choose(q, [c, -s, -c, s])
    return sin, cos


def _block(rows, block, salt, seed):
    rows = _u64(rows)
    return philox4x32_10(rows & _MASK32, rows >> np.uint64(32), block, salt, seed)


def normal2(words):
    """Box-Muller of one block: (n0, n1, rad) with rad = sqrt(-2 log u) (the normals' scale,
    which bounds their rounding error)."""
    u, v = u01(words[0], words[1]), u01(words[2], words[3])
    rad = np.sqrt(-2.0 * np.log(u))
    s, c = sincospi(2.0 * v)
    return rad * c, rad * s, rad


def rows_of(B, offset):
    return np.uint64(offset) + np.arange(B, dtype=np.uint64)


# ------------------------------------------------------------------------------ MA2
def prior_ma2(B, seed, offset=0, mode=0, t1=None):
    """prior_ma2_kernel: one block (row, row >> 32, 0, salt) -> u (t1, triangular on [-2, 2]) and
    v (t2 uniform on [max(-1 - t1, -1 + t1), 1]).  mode 0: both, 1: t1 only, 2: t2 given t1."""
    if mode == 2:
        t1 = np.asarray(t1, dtype=np.float64).reshape(-1)
        B = t1.size
    w = _block(rows_of(B, offset), 0, SALT_PRIOR_MA2, seed)
    u, v = u01(w[0], w[1]), u01(w[2], w[3])
    if mode != 2:
        with np.errstate(invalid='ignore'):
            t1 = np.where(u < 0.5, np.sqrt(2.0 * u) * 2.0 - 2.0, -np.sqrt(2.0 * (1.0 - u)) * 2.0 + 2.0)
    if mode == 1:
        return t1, None
    loc = np.maximum(-1.0 - t1, -1.0 + t1)
    return t1, loc + (1.0 - loc) * v


def ma2_innovations(B, n_obs, seed, offset=0):
    """The n_obs + 2 innovations w of each row of sim_ma2_kernel and their Box-Muller radii:
    block 0 gives w_0, w_1; block 1 + k0/2 + q gives w_{k0 + 2 + 2q}, w_{k0 + 3 + 2q}, i.e. block m
    gives (w_{2m}, w_{2m+1})."""
    nb = (n_obs + 3) // 2
    rows = rows_of(B, offset)[:, None]
    m = np.arange(nb, dtype=np.uint64)[None, :]
    n0, n1, rad = normal2(_block(rows, m, SALT_SIM_MA2, seed))
    w = np.empty((B, 2 * nb))
    r = np.empty((B, 2 * nb))
    w[:, 0::2], w[:, 1::2] = n0, n1
    r[:, 0::2], r[:, 1::2] = rad, rad
    return w[:, :n_obs + 2], r[:, :n_obs + 2]


def sim_ma2(t1, t2, n_obs, seed, offset=0):
    """MA2 data X (B, n_obs): x_k = (w_{k+2} + t1 w_{k+1}) + t2 w_k, each step rounded, and a bound
    of the replay's error per element (from the normals' error 1e-14 max(1, rad))."""
    t1 = np.asarray(t1, dtype=np.float64).reshape(-1, 1)
    t2 = np.asarray(t2, dtype=np.float64).reshape(-1, 1)
    w, rad = ma2_innovations(t1.shape[0], n_obs, seed, offset)
    X = (w[:, 2:] + t1 * w[:, 1:-1]) + t2 * w[:, :-2]
    e = 1e-14 * np.maximum(1.0, rad)
    err = e[:, 2:] + np.abs(t1) * e[:, 1:-1] + np.abs(t2) * e[:, :-2] + 4 * 2.0 ** -52 * (
        np.abs(w[:, 2:]) + np.abs(t1 * w[:, 1:-1]) + np.abs(t2 * w[:, :-2]))
    return X, err


# ------------------------------------------------------------------------------ Gaussian model
def sim_gauss(mu, sigma, n_obs, seed, offset=0):
    """sim_gauss_kernel: block m = k0/2 + q gives z_{2m}, z_{2m+1}; y = mu + sigma z.  Returns
    (Y, bound of the replay's error per element)."""
    mu = np.asarray(mu, dtype=np.float64).reshape(-1, 1)
    sigma = np.asarray(sigma, dtype=np.float64).reshape(-1, 1)
    B, nb = mu.shape[0], (n_obs + 1) // 2
    m = np.arange(nb, dtype=np.uint64)[None, :]
    n0, n1, rad = normal2(_block(rows_of(B, offset)[:, None], m, SALT_SIM_GAUSS, seed))
    z = np.empty((B, 2 * nb))
    r = np.empty((B, 2 * nb))
    z[:, 0::2], z[:, 1::2] = n0, n1
    r[:, 0::2], r[:, 1::2] = rad, rad
    z, r = z[:, :n_obs], r[:, :n_obs]
    Y = mu + sigma * z
    err = np.abs(sigma) * 1e-14 * np.maximum(1.0, r) + 4 * 2.0 ** -52 * (np.abs(mu) + np.abs(sigma * z))
    return Y, err


def _ndtri(p):
    from scipy.special import ndtri
    return ndtri(p)


def gauss_prior_constants(prm):
    """The constants make_gauss_prior passes to the kernels: sigma ~ truncnorm(a, b) is drawn by
    inverse-CDF sampling of the interval [lo, hi] = [a, b] (a <= 0) or, in the upper tail
    (a > 0), of its mirror image [-b, -a] with the sign flipped afterwards, so that the CDF values
    stay small and accurate.  Returns (lo, hi, sign, cdf_lo, mass)."""
    from scipy.special import erfc
    a, b = float(prm[2]), float(prm[3])
    flip = a > 0
    lo, hi = (-b, -a) if flip else (a, b)
    r2 = 0.7071067811865476
    cdf_lo = 0.5 * erfc(-lo * r2)
    mass = 0.5 * erfc(-hi * r2) - cdf_lo
    return lo, hi, (-1.0 if flip else 1.0), cdf_lo, mass


def prior_gauss(B, seed, prm, offset=0):
    """prior_gauss_kernel: one block (row, row >> 32, 0, salt); mu = mu_lo + mu_w u,
    sigma = sign * clamp(ndtri(cdf_lo + v mass), lo, hi)."""
    w = _block(rows_of(B, offset), 0, SALT_PRIOR_GAUSS, seed)
    u, v = u01(w[0], w[1]), u01(w[2], w[3])
    lo, hi, sign, cdf_lo, mass = gauss_prior_constants(prm)
    mu = prm[0] + prm[1] * u
    sigma = sign * np.minimum(np.maximum(_ndtri(cdf_lo + v * mass), lo), hi)
    return mu, sigma


# ------------------------------------------------------------------------------ g-and-k
def gnk_quantile(A, B, g, k, c, z):
    """gnkmath.cuh's operation order."""
    e = np.exp(-g * z)
    skew = 1.0 + c * ((1.0 - e) / (1.0 + e))
    kurt = (1.0 + z * z) ** k
    return A + ((B * skew) * kurt) * z


def sim_gnk(A, Bs, g, k, c, n_obs, seed, offset=0):
    """sim_gnk_kernel: block q of a row gives the normals of observations 2q, 2q + 1.  Returns
    (Y, bound of the replay's error per element): rtol 1e-12 of the terms, plus the normals' error
    1e-14 max(1, rad) times a bound of |dQ/dz|."""
    cols = [np.asarray(v, dtype=np.float64).reshape(-1, 1) for v in (A, Bs, g, k)]
    A, Bs, g, k = cols
    B, nb = A.shape[0], (n_obs + 1) // 2
    q = np.arange(nb, dtype=np.uint64)[None, :]
    n0, n1, rad = normal2(_block(rows_of(B, offset)[:, None], q, SALT_SIM_GNK, seed))
    z = np.empty((B, 2 * nb))
    r = np.empty((B, 2 * nb))
    z[:, 0::2], z[:, 1::2] = n0, n1
    r[:, 0::2], r[:, 1::2] = rad, rad
    z, r = z[:, :n_obs], r[:, :n_obs]
    Y = gnk_quantile(A, Bs, g, k, c, z)
    kurt = (1.0 + z * z) ** k
    slope = np.abs(Bs) * (1.0 + abs(c)) * kurt * (1.0 + 2.0 * np.abs(k) + np.abs(g * z))
    err = 1e-12 * (np.abs(A) + np.abs(Y - A)) + slope * 1e-14 * np.maximum(1.0, r)
    return Y, err


# ------------------------------------------------------------------------------ mixture proposals
def _cumsum_tiles(w, n, width):
    v = np.ones(n) if w is None else np.asarray(w, dtype=np.float64).reshape(-1)
    pad = (-n) % width
    return np.concatenate([v, np.zeros(pad)]).reshape(-1, width)


def _warp_inclusive_scan(x):
    """Hillis-Steele scan of __shfl_up_sync steps 1, 2, 4, 8, 16 over the last axis (32 lanes)."""
    incl = x.copy()
    for o in (1, 2, 4, 8, 16):
        t = incl[..., :-o].copy()
        incl[..., o:] = incl[..., o:] + t
    return incl


def _sequential_prefix(x):
    """prefix[w] = ((0 + x_0) + x_1) + ... + x_{w-1}, summed left to right (exclusive)."""
    out = np.zeros_like(x)
    acc = np.zeros(x.shape[:-1])
    for j in range(x.shape[-1] - 1):
        acc = acc + x[..., j]
        out[..., j + 1] = acc
    return out


def gm_cdf_warp_scan(w, n):
    """The summation order of the cumsum_kernel this project had before the monotone scan: tiles of
    1024, a warp shuffle scan per warp, warp totals added left to right, out = (carry + woff) + incl.
    Kept to show that this order can make the table decrease where a weight is zero."""
    tiles = _cumsum_tiles(w, n, 1024)
    out = np.empty(tiles.shape)
    carry = 0.0
    for t, tile in enumerate(tiles):
        incl = _warp_inclusive_scan(tile.reshape(32, 32))
        woff = _sequential_prefix(incl[:, 31])
        o = (carry + woff[:, None]) + incl
        out[t] = o.reshape(-1)
        carry = o[31, 31]
    return out.reshape(-1)[:n]


GM_CDF_PER_THREAD = 8


def gm_cdf(w, n=None):
    """cumsum_kernel's order of additions (one block of 1024 threads, GM_CDF_PER_THREAD consecutive
    elements per thread and tile): sequential sums per thread, a warp shuffle scan of the thread
    totals, warp totals added left to right, base = carry + (woff + exclusive); then the running
    sums from that base, and a running maximum over the threads' last values so the table cannot
    decrease (a thread's leading zero weights take that maximum, i.e. the entry before them).  The
    result is the device's table bit for bit (only additions and maxima)."""
    K = GM_CDF_PER_THREAD
    n = int(np.asarray(w).size) if w is not None else int(n)
    tiles = _cumsum_tiles(w, n, 1024 * K)
    out = np.empty(tiles.shape)
    carry = 0.0
    for t, tile in enumerate(tiles):
        v = tile.reshape(32, 32, K)                  # warp, lane, element
        tot = v[..., 0].copy()
        for j in range(1, K):
            tot = tot + v[..., j]
        incl = _warp_inclusive_scan(tot)
        excl = np.zeros_like(incl)
        excl[:, 1:] = incl[:, :-1]
        woff = _sequential_prefix(incl[:, 31])
        run = carry + (woff[:, None] + excl)
        r = np.empty_like(v)
        seen = np.zeros(run.shape, dtype=bool)
        for j in range(K):
            run = run + v[..., j]
            seen = seen | (v[..., j] != 0.0)
            r[..., j] = np.where(seen, run, -np.inf)
        last = r[..., K - 1].reshape(-1)
        pm = np.maximum.accumulate(np.concatenate([[carry], last[:-1]]))
        o = np.maximum(r.reshape(1024, K), pm[:, None])
        out[t] = o.reshape(-1)
        carry = o[-1, -1]
    return out.reshape(-1)[:n]


def _first_ge(cumw, u):
    """cumsum lookup exactly as gm_rvs_kernel's binary search (first index with cumw >= u on a
    sorted table; the same probe sequence on any table)."""
    lo = np.zeros(u.shape, dtype=np.int64)
    hi = np.full(u.shape, cumw.size - 1, dtype=np.int64)
    while True:
        act = lo < hi
        if not act.any():
            return lo
        mid = (lo + hi) >> 1
        below = cumw[mid] < u
        lo = np.where(act & below, mid + 1, lo)
        hi = np.where(act & ~below, mid, hi)


def _support_margin(x, support, box):
    """(inside, distance to the nearest support boundary) of draws x (rows, p)."""
    if support == 0:
        return np.ones(x.shape[0], dtype=bool), np.full(x.shape[0], np.inf)
    if support == 1:
        ax = np.abs(x[:, 0])
        inside = (ax < 2.0) & (x[:, 1] >= -1.0 + ax) & (x[:, 1] <= 1.0)
        margin = np.minimum.reduce([np.abs(2.0 - ax), np.abs(x[:, 1] + 1.0 - ax), np.abs(1.0 - x[:, 1])])
        return inside, margin
    lo, hi = np.asarray(box[0], dtype=np.float64), np.asarray(box[1], dtype=np.float64)
    inside = np.all((x >= lo) & (x <= hi), axis=1)
    margin = np.min(np.minimum(np.abs(x - lo), np.abs(hi - x)), axis=1)
    return inside, margin


def gm_rvs(means, L, cumw, B, seed, offset=0, support=0, box=None, max_trials=1000):
    """gm_rvs_kernel.  Trial t of a row: block 4t -> u = u01 * cumw[-1] -> component (first index
    with cumw >= u, the kernel's binary search on the given table); block 4t + 1 -> z_0, z_1; block
    4t + 2 -> z_2, z_3 (p > 2 only); x_a = means[c, a] + sum_{b <= a} L[a, b] z_b accumulated for
    b = 0 .. a; accepted when inside the support; after max_trials failures the last draw is kept.

    Returns (x (B, p), trial (B,) accepted trial or -1 when none was, component (B,),
    err (B,) bound of the replay's error per row, margin (B,) the smallest distance of any draw up
    to the deciding trial from a support boundary)."""
    means = np.asarray(means, dtype=np.float64)
    L = np.asarray(L, dtype=np.float64)
    cumw = np.asarray(cumw, dtype=np.float64)
    p = means.shape[1]
    total = cumw[-1]
    rows = rows_of(B, offset)
    x = np.zeros((B, p))
    err = np.zeros(B)
    comp = np.zeros(B, dtype=np.int64)
    trial = np.full(B, -1, dtype=np.int64)
    margin = np.full(B, np.inf)
    act = np.arange(B)
    for t in range(max_trials):
        if act.size == 0:
            break
        r = rows[act]
        w = _block(r, 4 * t, SALT_GM_RVS, seed)
        c = _first_ge(cumw, u01(w[0], w[1]) * total)
        z = np.zeros((act.size, 4))
        rad = np.zeros((act.size, 2))
        z[:, 0], z[:, 1], rad[:, 0] = normal2(_block(r, 4 * t + 1, SALT_GM_RVS, seed))
        if p > 2:
            z[:, 2], z[:, 3], rad[:, 1] = normal2(_block(r, 4 * t + 2, SALT_GM_RVS, seed))
        zerr = 1e-14 * np.maximum(1.0, rad)[:, [0, 0, 1, 1]]
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
            et = np.maximum(et, e + 4 * 2.0 ** -52 * mag)
        inside, mg = _support_margin(xt, support, box)
        x[act], err[act], comp[act] = xt, et, c
        margin[act] = np.minimum(margin[act], mg)
        trial[act[inside]] = t
        act = act[~inside]
    return x, trial, comp, err, margin
