"""NumPy replay of the scratch assay streams (elfi_b200/csrc/scratch_assay.cuh) -- TEST
INFRASTRUCTURE ONLY.

Built on oracle/streams.py (the Philox generator and u01): slot s of phase f (0 motility,
1 proliferation) in iteration t of a row uses the block (x, y, z, w) of counter (row, row >> 32,
2 t + f, SALT_SCRATCH + s); the slot is kept when 1 - u01(x, y) < p, picks list index
((z << 32 | w) * n) >> 64 and direction y & 3.  Every decision is an integer or exact fp64
comparison, so the replay reproduces every lattice bit of the device and of the header's host
build.  The law is stated in the header; here it is restated in NumPy, one row at a time for the
motility moves (they depend on each other in slot order), vectorised elsewhere.
"""
import numpy as np

import streams

SALT_SCRATCH = 0x53434131
MASK32 = np.uint64(0xFFFFFFFF)


def mulhi_n(z, w, n):
    """((z << 32 | w) * n) >> 64 for 32-bit words z, w and n < 2^32, exactly in uint64."""
    z, w, n = (np.asarray(v, dtype=np.uint64) for v in (z, w, n))
    return ((z * n + ((w * n) >> np.uint64(32))) >> np.uint64(32)).astype(np.int64)


def targets(sites, dirs, nrows, ncols):
    """Sites reached from `sites` in directions `dirs` (0: row + 1, 1: row - 1, 2: col + 1,
    3: col - 1), clamped to the grid."""
    r, c = np.divmod(np.asarray(sites, dtype=np.int64), ncols)
    dirs = np.asarray(dirs)
    r = np.where(dirs == 0, np.minimum(r + 1, nrows - 1), np.where(dirs == 1, np.maximum(r - 1, 0), r))
    c = np.where(dirs == 2, np.minimum(c + 1, ncols - 1), np.where(dirs == 3, np.maximum(c - 1, 0), c))
    return r * ncols + c


def slots(row, t, f, n, p, seed):
    """(kept, index, direction) of the n slots of phase f in iteration t of row `row`."""
    s = np.arange(n, dtype=np.uint64)
    w = streams._block(np.uint64(row), np.uint64(2 * t + f), np.uint64(SALT_SCRATCH) + s, seed)
    kept = 1.0 - streams.u01(w[0], w[1]) < p
    return kept, mulhi_n(w[2], w[3], n), (w[1] & np.uint64(3)).astype(np.int64)


def steps(obs_period=12, obs_interval=1 / 12, tau=1 / 24):
    num_iter = int(obs_period / tau)
    interval = int(obs_interval / tau)
    return num_iter, interval, int(num_iter / interval)


def sim(P, init, num_obs, interval, seed, offset=0):
    """(X (B, nrows, ncols, num_obs + 1) uint8, S (B, num_obs + 1) float64) of parameters P (B, 2)
    from the lattice init (nrows, ncols), rows offset + i."""
    P = np.asarray(P, dtype=np.float64).reshape(-1, 2)
    init = np.asarray(init) != 0
    nrows, ncols = init.shape
    N = nrows * ncols
    B = P.shape[0]
    X = np.empty((B, N, num_obs + 1), dtype=np.uint8)
    rows = streams.rows_of(B, offset)
    for b in range(B):
        pm, pp = P[b]
        lat = init.reshape(-1).copy()
        X[b, :, 0] = lat
        full = False
        for t in range(num_obs * interval):
            if not full:
                cells = np.flatnonzero(lat)
                n = cells.size
                full = n == N
            if not full:
                if pm > 0:
                    kept, idx, dirs = slots(rows[b], t, 0, n, pm, seed)
                    for i, d in zip(idx[kept], dirs[kept]):
                        frm = cells[i]
                        to = targets(frm, d, nrows, ncols)
                        if not lat[to]:
                            lat[frm], lat[to] = False, True
                            cells[i] = to
                if pp > 0:
                    kept, idx, dirs = slots(rows[b], t, 1, n, pp, seed)
                    lat[targets(cells[idx[kept]], dirs[kept], nrows, ncols)] = True
            if (t + 1) % interval == 0:
                X[b, :, (t + 1) // interval] = lat
    X = X.reshape(B, nrows, ncols, num_obs + 1)
    return X, summaries(X)


def summaries(X):
    """The mismatches between consecutive frames and the cells of the last frame, (B, F)."""
    X = np.asarray(X) != 0
    ds = np.sum(X[..., :-1] != X[..., 1:], axis=(1, 2))
    return np.concatenate([ds, np.sum(X[..., -1], axis=(1, 2))[:, None]], axis=1).astype(np.float64)
