"""NumPy replay of the toad simulator's stream and step (elfi_b200/csrc/toad.cu) -- TEST
INFRASTRUCTURE ONLY.

Built on oracle/streams.py (the Philox generator and u01).  Toad k on day d of a row uses the cell
c = d * n_toads + k: block (c << 1) | 0 gives the return uniform 1 - u01(x, y) and the refuge word
(z << 32) | w, block (c << 1) | 1 gives TH = (1 - u01(x, y)) pi - pi / 2 and W = -log(u01(z, w)).
The uniforms, the return decisions and the refuge days are exact.  The step is SciPy's levy_stable
formula (beta = 0) in NumPy; it differs from the device's only through the ulps of sin, cos, tan,
pow and log, and step_bound carries those through the formula with the condition numbers of its
two sums (see step_bound).
"""
import numpy as np

import streams

SALT_TOAD = 0x544F4144
EPS = 2.0 ** -52
U32 = np.uint64(32)


def draws(B, n_toads, n_days, seed, offset=0):
    """(u_ret, word, u_th, u_w), each (B, n_days - 1, n_toads): the draws of days 1 .. n_days - 1."""
    rows = streams.rows_of(B, offset)[:, None, None]
    d = np.arange(1, n_days, dtype=np.uint64)[None, :, None]
    k = np.arange(n_toads, dtype=np.uint64)[None, None, :]
    cell = d * np.uint64(n_toads) + k
    w0 = streams._block(rows, cell << np.uint64(1), SALT_TOAD, seed)
    w1 = streams._block(rows, (cell << np.uint64(1)) | np.uint64(1), SALT_TOAD, seed)
    u_ret = 1.0 - streams.u01(w0[0], w0[1])
    word = (w0[2] << U32) | w0[3]
    return u_ret, word, 1.0 - streams.u01(w1[0], w1[1]), streams.u01(w1[2], w1[3])


def refuge_day(word, d):
    """The high 64 bits of word * d (d < 2^31), exactly, in uint64 arithmetic."""
    word = np.asarray(word, dtype=np.uint64)
    d = np.asarray(d, dtype=np.uint64)
    lo, hi = word & np.uint64(0xFFFFFFFF), word >> U32
    return ((hi * d + ((lo * d) >> U32)) >> U32).astype(np.int64)


def step(alpha, gamma, u_th, u_w):
    """levy_stable.rvs(alpha, beta=0, scale=gamma) from the uniforms, in SciPy's order; returns the
    step and the condition numbers (|a| + |b|) / |a + b| of its two sums."""
    with np.errstate(all='ignore'):
        TH = u_th * np.pi + (-np.pi / 2)
        W = -np.log(u_w) * 1.0 + 0.0
        aTH = alpha * TH
        cosTH, tanTH = np.cos(TH), np.tan(TH)
        t1, t2 = cosTH / np.tan(aTH), np.sin(TH)
        s1, s2 = np.cos(aTH), np.sin(aTH) * tanTH
        den, num = t1 + t2, s1 + s2
        val = W / den * (num / W) ** (1.0 / alpha)
        bTH = 0.0 * TH
        v1 = 2 / np.pi * ((np.pi / 2 + bTH) * tanTH
                          - 0 * np.log((np.pi / 2 * W * cosTH) / (np.pi / 2 + bTH)))
        val = np.where(alpha == 1, v1, val)
        x = val * gamma + 0.0
        x = np.where(alpha == 1, x + 0 * gamma * np.log(gamma) / np.pi, x)
        c1 = np.where(alpha == 1, 1.0, (np.abs(t1) + np.abs(t2)) / np.abs(den))
        c2 = np.where(alpha == 1, 1.0, (np.abs(s1) + np.abs(s2)) / np.abs(num))
    return x, c1, c2


def step_bound(x, alpha, c1, c2, r=4 * EPS):
    """|device step - replayed step| bound: every sin, cos, tan, pow and log may differ by r
    (relative) between CUDA and NumPy; the sums amplify their inputs' errors by c1 (denominator)
    and c2 (numerator), pow by its exponent 1 / alpha <= 1."""
    rel_den = c1 * (2 * r + EPS) + EPS
    rel_num = c2 * (2 * r + EPS) + EPS
    rel = r + rel_den + EPS + (rel_num + r + EPS) / alpha + r + 2 * EPS
    return 2.0 * rel * np.abs(x)
