"""NumPy replay of the ARCH(1) streams (elfi_b200/csrc/arch.cu) -- TEST INFRASTRUCTURE ONLY.

Built on oracle/streams.py (the Philox generator, u01 and Box-Muller): block m of a row gives the
normals z_{2m}, z_{2m+1}, z_0 = e_0 and z_k = xi_k.  The replayed normals are within 1e-14 max(1,
rad) of the device's (streams.py), so the series is compared within a bound carried through the
recurrence to first order, plus the roundings of every step.
"""
import numpy as np

import streams

SALT_ARCH = 0x41524348
EPS = 2.0 ** -52


def normals(B, n_obs, seed, offset=0):
    """(z, rad) of shape (B, n_obs + 1): z[:, k] as arch.cu draws it and its Box-Muller radius."""
    nb = n_obs // 2 + 1
    rows = streams.rows_of(B, offset)[:, None]
    m = np.arange(nb, dtype=np.uint64)[None, :]
    n0, n1, rad = streams.normal2(streams._block(rows, m, SALT_ARCH, seed))
    z = np.empty((B, 2 * nb))
    r = np.empty((B, 2 * nb))
    z[:, 0::2], z[:, 1::2] = n0, n1
    r[:, 0::2], r[:, 1::2] = rad, rad
    return z[:, :n_obs + 1], r[:, :n_obs + 1]


def sim_arch(P, n_obs, seed, offset=0):
    """(Y (B, n_obs), err (B, n_obs)): the kernel's recurrence on the replayed normals and a bound
    of the replay's error per element.  Needs t2 >= 0 (then sqrt(0.2 + t2 e^2) >= sqrt(0.2))."""
    P = np.asarray(P, dtype=np.float64)
    t1, t2 = P[:, 0], P[:, 1]
    B = P.shape[0]
    z, rad = normals(B, n_obs, seed, offset)
    dz = 1e-14 * np.maximum(1.0, rad)
    Y = np.empty((B, n_obs))
    err = np.empty((B, n_obs))
    e, de = z[:, 0], dz[:, 0]
    y, dy = np.zeros(B), np.zeros(B)
    for k in range(1, n_obs + 1):
        s = np.sqrt(0.2 + t2 * (e * e))
        e_new = z[:, k] * s
        # d(xi s) = s dxi + |xi| t2 |e| de / s, plus the four roundings of the step
        de = s * dz[:, k] + np.abs(z[:, k]) * t2 * np.abs(e) * de / s + 4 * EPS * np.abs(e_new) + \
            np.abs(z[:, k]) * 2 * EPS * s
        e = e_new
        y_new = t1 * y + e
        dy = np.abs(t1) * dy + de + 2 * EPS * (np.abs(t1 * y) + np.abs(y_new))
        y = y_new
        Y[:, k - 1] = y
        err[:, k - 1] = 4 * dy
    return Y, err
