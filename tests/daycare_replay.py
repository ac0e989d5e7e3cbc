"""NumPy replay of the day care simulator (elfi_b200/csrc/daycare.cu, arithmetic in daycare.cuh) --
TEST INFRASTRUCTURE ONLY.

Built on oracle/streams.py (the Philox generator and u01).  Row i = offset + i; transition k of DCC
c uses block k of salt SALT_DAYCARE + c: E = -log(u01(x, y)) and the uniform 1 - u01(z, w).  The
uniforms, the hazards, the total, the selection and the state are exact restatements (NumPy rounds
each elementwise operation once, and a running sum along an axis is np.cumsum's left-to-right
order); only E (NumPy's log against the device's) may differ by an ulp, and with it the times.  A
time can therefore decide a different K only where it lies within a few ulps of time_end, so the
replay reports, per row, the smallest relative distance of any DCC's time from time_end.
"""
import numpy as np

import streams

SALT_DAYCARE = 0x44434300


def lcm_upto(n):
    L = 1
    for k in range(2, n + 1):
        L = L * k // np.gcd(L, k)
    return L


def _bits(mask, n_strains):
    return ((mask[:, :, None] >> np.arange(n_strains, dtype=np.uint64)) & np.uint64(1)).astype(bool)


def _nth(member, j):
    """Index of the j-th True of each row of member (j < count)."""
    c = np.cumsum(member, axis=1)
    return np.argmax(member & (c == (j + 1)[:, None]), axis=1)


def row_ok(P, f, n_ind, n_strains, time_end):
    """dc_row_ok: t1, t2, t3 finite and >= 0, and time_end n_ind n_strains times the largest cell
    hazard below 2^32 - 1."""
    P = np.asarray(P, dtype=np.float64)
    with np.errstate(invalid='ignore', over='ignore'):
        fin = np.all(np.isfinite(P) & (P >= 0), axis=1)
        h = (P[:, 0] + 1e-9) + P[:, 1] * np.max(f)
        cell = np.fmax(1.0, np.fmax(1.0, P[:, 2]) * h)
        return fin & (time_end * float(n_ind) * float(n_strains) * cell < 4294967295.0)


def simulate(P, n_dcc, n_ind, n_strains, f, n_obs, time_end, seed, offset=0):
    """(masks (B, n_dcc, n_ind) uint64, K (B,), k_c (B, n_dcc), margin (B,)) of the kernel for
    parameters P (B, 3); rows that row_ok refuses give K = -1 and empty masks."""
    P = np.asarray(P, dtype=np.float64)
    f = np.asarray(f, dtype=np.float64)
    B = P.shape[0]
    N = B * n_dcc
    L = lcm_upto(n_strains)
    Lk = np.zeros(n_strains + 1, dtype=np.int64)
    Lk[1:] = [L // k for k in range(1, n_strains + 1)]
    Ld, nf = float(L), 1.0 / (n_ind - 1)
    rows = np.repeat(streams.rows_of(B, offset), n_dcc)
    dcc = np.tile(np.arange(n_dcc, dtype=np.uint64), B)
    t1, t2, t3 = (np.repeat(P[:, j], n_dcc)[:, None] for j in range(3))
    valid_row = row_ok(P, f, n_ind, n_strains, time_end)
    mask = np.zeros((N, n_ind), dtype=np.uint64)
    num = np.zeros((N, n_strains), dtype=np.int64)
    cnt = np.zeros((N, n_strains), dtype=np.int64)
    n_free = np.full(N, n_ind, dtype=np.int64)
    t = np.zeros(N)
    K = np.where(valid_row, 0, -1).astype(np.int64)
    k_c = np.zeros(N, dtype=np.int64)
    margin = np.full(B, np.inf)
    pc = t2 * f[None, :]
    running = valid_row.copy()
    k = 0
    while running.any():
        lanes = np.repeat(running, n_dcc)
        idx = np.nonzero(lanes)[0]
        w = streams.philox4x32_10(rows[idx] & np.uint64(0xFFFFFFFF), rows[idx] >> np.uint64(32), k,
                                  np.uint64(SALT_DAYCARE) + dcc[idx], seed)
        E = -np.log(streams.u01(w[0], w[1]))
        x = 1.0 - streams.u01(w[2], w[3])
        Es = num[idx].astype(np.float64) / Ld
        h = ((t1[idx] * Es) * nf + 1e-9) + pc[idx]
        c = cnt[idx]
        fr = n_free[idx][:, None]
        m = n_ind - fr - c
        W = c.astype(np.float64) + h * (fr.astype(np.float64) + t3[idx] * m.astype(np.float64))
        cum = np.cumsum(W, axis=1)
        H = cum[:, -1]
        target = x * H
        pos = W > 0
        hit = pos & (target[:, None] < cum)
        first = np.argmax(hit, axis=1)
        last = n_strains - 1 - np.argmax(pos[:, ::-1], axis=1)
        s = np.where(hit.any(axis=1), first, last)
        ar = np.arange(idx.size)
        start = np.where(s > 0, cum[ar, np.maximum(s - 1, 0)], 0.0)
        hs, cs, ms = h[ar, s], c[ar, s], m[ar, s]
        frs = n_free[idx]
        t3i = t3[idx, 0]
        w0 = cs.astype(np.float64)
        w1 = hs * frs.astype(np.float64)
        th = t3i * hs
        w2 = th * ms.astype(np.float64)

        def clamp0(v):
            return np.where(v > 0, v, 0.0)

        def slot(q, n):
            return np.where(q > 0, np.where(q >= (n - 1).astype(np.float64), n - 1,
                                            np.floor(np.where(q > 0, np.minimum(q, 2.0 ** 62), 0))
                                            .astype(np.int64)), 0)
        r = clamp0(target - start)
        cat0 = (w0 > 0) & ((r < w0) | ~((w1 > 0) | (w2 > 0)))
        r1 = clamp0(r - w0)
        cat1 = ~cat0 & (w1 > 0) & ((r1 < w1) | ~(w2 > 0))
        r2 = clamp0(r1 - w1)
        with np.errstate(divide='ignore', invalid='ignore'):
            j = np.where(cat0, slot(r, cs), np.where(cat1, slot(r1 / hs, frs), slot(r2 / th, ms)))
        mk = mask[idx]
        bit = np.uint64(1) << s.astype(np.uint64)
        has = (mk & bit[:, None]) != 0
        member = np.where(cat0[:, None], has,
                          np.where(cat1[:, None], mk == 0, (mk != 0) & ~has))
        child = _nth(member, j)
        # flip strain s of the child
        old = mk[ar, child]
        b_old = _bits(old[:, None], n_strains)[:, 0]
        n_old = b_old.sum(axis=1)
        new = old ^ bit
        b_new = _bits(new[:, None], n_strains)[:, 0]
        n_new = b_new.sum(axis=1)
        num[idx] += b_new * Lk[n_new][:, None] - b_old * Lk[n_old][:, None]
        cnt[idx, s] += np.where(b_old[ar, s], -1, 1)
        n_free[idx] += (new == 0).astype(np.int64) - (old == 0).astype(np.int64)
        mask[idx, child] = new
        before = t[idx] < time_end
        t[idx] = t[idx] + (1.0 / H) * E
        k_c[idx] = np.where(before & (t[idx] >= time_end), k + 1, k_c[idx])
        rel = np.abs(t[idx] - time_end) / time_end
        row_of = idx // n_dcc
        np.minimum.at(margin, row_of, rel)
        k += 1
        K[running] = k
        running = running & ~(t.reshape(B, n_dcc) >= time_end).all(axis=1)
    return mask.reshape(B, n_dcc, n_ind), K, k_c.reshape(B, n_dcc), margin


def data_of(masks, n_obs, n_strains):
    """(B, n_dcc, n_obs, n_strains) bool data of the first n_obs children."""
    m = masks[:, :, :n_obs]
    return ((m[..., None] >> np.arange(n_strains, dtype=np.uint64)) & np.uint64(1)).astype(bool)
