"""NumPy replay of the M/G/1 streams (elfi_b200/csrc/mg1.cu) -- TEST INFRASTRUCTURE ONLY.

Built on oracle/streams.py (the Philox generator and u01): block j of a row gives u = u01(x, y)
for the inter-arrival time and u' = u01(z, w) for the service time.  U = t1 + (t2 - t1) u' is
replayed exactly; W = (1 / t3)(-log u) within the ulps of log; the series within a bound carried
through the recurrence (the max is 1-Lipschitz, so the errors of the sums add up).
"""
import numpy as np

import streams

SALT_MG1 = 0x4D473151
EPS = 2.0 ** -52


def uniforms(B, n, seed, offset=0):
    """(u, v) of shape (B, n): the inter-arrival and service uniforms of mg1.cu."""
    rows = streams.rows_of(B, offset)[:, None]
    j = np.arange(n, dtype=np.uint64)[None, :]
    w = streams._block(rows, j, SALT_MG1, seed)
    return streams.u01(w[0], w[1]), streams.u01(w[2], w[3])


def sim_mg1(P, n, seed, offset=0):
    """(Y (B, n), err (B, n), W, U): the kernel's recurrence on the replayed draws and a bound of
    the replay's error per element (finite rows)."""
    P = np.asarray(P, dtype=np.float64)
    B = P.shape[0]
    u, v = uniforms(B, n, seed, offset)
    with np.errstate(all='ignore'):
        inv = 1 / P[:, 2]
        rng = P[:, 1] - P[:, 0]
        W = inv[:, None] * -np.log(u)
        U = P[:, 0, None] + rng[:, None] * v
        Y = np.empty((B, n))
        err = np.empty((B, n))
        sw, sx = np.zeros(B), np.zeros(B)
        dsw, dsx = np.zeros(B), np.zeros(B)
        for j in range(n):
            sw = sw + W[:, j]
            dsw = dsw + 4 * EPS * np.abs(W[:, j]) + 2 * EPS * np.abs(sw)
            d = sw - sx
            m = np.where(d < 0, 0.0, d)
            y = U[:, j] + m
            dy = dsw + dsx + 2 * EPS * (np.abs(d) + np.abs(y))
            sx = sx + y
            # sx + y = max(sx, sw) + U: the errors of sx and sw do not add up in the new sum
            dsx = np.maximum(dsx, dsw) + 2 * EPS * (np.abs(d) + np.abs(y) + np.abs(sx))
            Y[:, j] = y
            err[:, j] = 2 * dy
    bad = (np.signbit(inv) & ~np.isnan(inv)) | ~np.isfinite(rng)
    Y[bad] = np.nan
    return Y, err, W, U
