"""NumPy replay of the Lotka-Volterra simulator (elfi_b200/csrc/lotka_volterra.cu) -- TEST
INFRASTRUCTURE ONLY.

Built on oracle/streams.py (the Philox generator, u01 and Box-Muller).  Row i = offset + i; event k
uses block k of salt SALT_LV: E = -log(u01(x, y)) and the reaction uniform 1 - u01(z, w);
observation j uses block j of salt SALT_LV_NOISE, whose Box-Muller pair times sigma is the prey and
predator noise.  The uniforms and every hazard, probability and reaction are exact; only E (NumPy's
log against the device's) and the normals may differ by an ulp.  Such a difference can change the
result only where an event time lies on a grid time or on time_end, or where a noisy value lies on
an integer, so the replay reports, per row, the smallest relative distance of any event time from
the grid times and time_end, and of any noisy value from an integer.
"""
import numpy as np

import streams

SALT_LV = 0x4C4F5456
SALT_LV_NOISE = 0x4C564E4F
INT32_LOW, INT32_HIGH = -2147483649.0, 2147483648.0


def to_int32(v):
    """NumPy's float64 -> int32 cast on x86-64, as float64."""
    v = np.asarray(v, dtype=np.float64)
    with np.errstate(invalid='ignore'):
        ok = (v > INT32_LOW) & (v < INT32_HIGH)
        return np.where(ok, np.trunc(np.where(ok, v, 0.0)), -2147483648.0)


def _grid_margin(t1, t_out):
    """Relative distance of each t1 from the nearest positive grid time."""
    g = t_out[1:]
    i = np.clip(np.searchsorted(g, t1), 0, g.size - 1)
    lo = g[np.maximum(i - 1, 0)]
    hi = g[i]
    with np.errstate(invalid='ignore'):
        return np.minimum(np.abs(t1 - lo) / lo, np.abs(t1 - hi) / hi)


def simulate(P, n_obs, time_end, seed, offset=0, max_events=2 ** 20):
    """(obs (B, n_obs, 2), n_events (B,), margin (B,)) of the kernel for parameters P (B, 6)."""
    P = np.asarray(P, dtype=np.float64)
    B = P.shape[0]
    t_out = np.linspace(0, time_end, n_obs)
    rows = streams.rows_of(B, offset)
    r1, r2, r3, sigma = P[:, 0], P[:, 1], P[:, 2], P[:, 5]
    X, Y = np.floor(P[:, 3]), np.floor(P[:, 4])
    with np.errstate(invalid='ignore'):
        ok = ((r1 >= 0) & (r2 >= 0) & (r3 >= 0) & (sigma >= 0) & (X >= 0) & (X < 2 ** 31)
              & (Y >= 0) & (Y < 2 ** 31))
    obs = np.full((B, n_obs, 2), np.nan)
    obs[ok, 0, 0], obs[ok, 0, 1] = X[ok], Y[ok]
    t = np.zeros(B)
    k = np.zeros(B, dtype=np.int64)
    j = np.ones(B, dtype=np.int64)
    margin = np.full(B, np.inf)
    live = ok.copy()
    with np.errstate(all='ignore'):
        while True:
            run = live & (t < time_end) & (k < max_events)
            if not run.any():
                break
            i = np.nonzero(run)[0]
            w = streams._block(rows[i], k[i].astype(np.uint64), SALT_LV, seed)
            E = -np.log(streams.u01(w[0], w[1]))
            u = 1.0 - streams.u01(w[2], w[3])
            x0, y0 = X[i], Y[i]
            h1, h2, h3 = r1[i] * x0, (r2[i] * x0) * y0, r3[i] * y0
            tot = (h1 + h2) + h3
            inv = 1.0 / tot
            p1, p2 = h1 * inv, h2 * inv
            reaction = np.where(np.isinf(inv), 3, (u >= p1).astype(int) + (u >= p1 + p2))
            bad = ~(tot >= 0)
            x1 = x0 + np.where(reaction == 0, 1.0, np.where(reaction == 1, -1.0, 0.0))
            y1 = y0 + np.where(reaction == 1, 1.0, np.where(reaction == 2, -1.0, 0.0))
            t1 = np.where(y1 == 0, time_end, t[i] + inv * E)
            moved = (y1 != 0) & ~bad
            m = np.minimum(_grid_margin(t1, t_out), np.abs(t1 - time_end) / time_end)
            margin[i[moved]] = np.minimum(margin[i[moved]], m[moved])
            # emissions
            while True:
                jj = j[i]
                em = ~bad & (jj < n_obs) & (t1 >= t_out[np.minimum(jj, n_obs - 1)])
                if not em.any():
                    break
                e = np.nonzero(em)[0]
                r, je = i[e], jj[e]
                g = t_out[je]
                frac = (g - t[r]) / (t1[e] - t[r])
                n0, n1 = np.zeros(e.size), np.zeros(e.size)
                noisy = sigma[r] != 0
                if noisy.any():
                    a, b, _ = streams.normal2(streams._block(rows[r[noisy]], je[noisy].astype(np.uint64),
                                                             SALT_LV_NOISE, seed))
                    n0[noisy], n1[noisy] = sigma[r[noisy]] * a, sigma[r[noisy]] * b
                for s, (s0, s1, nz) in enumerate(((x0[e], x1[e], n0), (y0[e], y1[e], n1))):
                    v = ((s1 - s0) * frac + s0) + nz
                    obs[r, je, s] = to_int32(v)
                    if noisy.any():
                        dv = np.abs(v - np.round(v)) / np.maximum(1.0, np.abs(v))
                        margin[r[noisy]] = np.minimum(margin[r[noisy]], dv[noisy])
                j[r] += 1
            good = i[~bad]
            t[good], X[good], Y[good] = t1[~bad], x1[~bad], y1[~bad]
            k[good] += 1
            obs[i[bad]] = np.nan
            live[i[bad]] = False
    complete = live & (t >= time_end) & (j == n_obs)
    obs[~complete] = np.nan
    return obs, k, margin
