"""NumPy replay of the birth-death-mutation simulator (elfi_b200/csrc/bdm.cu) -- TEST
INFRASTRUCTURE ONLY.

Built on oracle/streams.py (the Philox generator and u01).  Row i = offset + i; event k uses block k
of salt SALT_BDM: u = 1 - u01(x, y) draws the event, v = 1 - u01(z, w) the cluster.  Every step is
exact (products of a uniform and a rate or an integer, sums of rates, integer counts), so the
replay equals the kernel row for row: counts and event counts.  The rows run together, one event
per live row per step.
"""
import numpy as np

import streams

SALT_BDM = 0x42444D31


def uniforms(rows, k, seed):
    """(u, v) of event k (array) of the counter rows (array)."""
    w = streams._block(rows, np.asarray(k).astype(np.uint64), SALT_BDM, seed)
    return 1.0 - streams.u01(w[0], w[1]), 1.0 - streams.u01(w[2], w[3])


def valid(P):
    a, d, t = (np.asarray(P, dtype=np.float64)[:, c] for c in range(3))
    with np.errstate(invalid='ignore', over='ignore'):
        total = ((0.0 + a) + d) + t
        return ((a >= 0) & (a < np.inf) & (d >= 0) & (d < np.inf) & (t >= 0) & (t < np.inf)
                & (total > 0) & (total < np.inf))


def simulate(P, N, seed, offset=0, max_events=2 ** 24):
    """(X (B, N) int16, n_events (B,) int64) of the kernel for rates P (B, 3)."""
    P = np.asarray(P, dtype=np.float64)
    B = P.shape[0]
    rows = streams.rows_of(B, offset)
    a, d, t = P[:, 0], P[:, 1], P[:, 2]
    ok = valid(P)
    with np.errstate(invalid='ignore', over='ignore'):
        total = ((0.0 + a) + d) + t
    c = np.zeros((B, N), dtype=np.int64)
    c[:, 0] = 1
    pop = np.ones(B, dtype=np.int64)
    k = np.zeros(B, dtype=np.int64)
    event = np.zeros(B, dtype=np.int64)
    cluster = np.zeros(B, dtype=np.int64)
    while True:
        run = ok & (pop > 0) & (pop < N + 1) & (k < max_events)
        if not run.any():
            break
        i = np.nonzero(run)[0]
        u, v = uniforms(rows[i], k[i], seed)
        x = u * total[i]
        cum0 = 0.0 + a[i]
        e = np.where(cum0 > x, 0, np.where(cum0 + d[i] > x, 1, 2))
        j = np.argmax(np.cumsum(c[i], axis=1) > (v * pop[i])[:, None], axis=1)
        c[i[e == 0], j[e == 0]] += 1
        c[i[e == 1], j[e == 1]] -= 1
        pop[i] += (e == 0).astype(np.int64) - (e == 1)
        mut = (e == 2) & (c[i, j] > 1)
        r = i[mut]
        c[r, j[mut]] -= 1
        z = np.argmax(c[r] == 0, axis=1)
        c[r, z] = 1
        event[i], cluster[i] = e, j
        k[i] += 1
    finished = ok & ~((pop > 0) & (pop < N + 1))
    undo = np.nonzero(finished & (event == 0))[0]
    c[undo, cluster[undo]] -= 1
    n_events = np.where(ok, k, -1)
    c[~finished] = -1
    return c.astype(np.int16), n_events
