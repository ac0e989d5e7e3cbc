"""NumPy replay of the AR(1) streams (elfi_b200/csrc/ar1.cu) -- TEST INFRASTRUCTURE ONLY.

Built on oracle/streams.py (the Philox generator, u01 and Box-Muller): block m of a row gives the
normals z_{2m}, z_{2m+1}, and z_k is the innovation of observation k + 1.  The replayed normals are
within 1e-14 max(1, rad) of the device's (streams.py), so the series is compared within a bound
carried through the recursion to first order, plus the roundings of every step.
"""
import numpy as np

import streams

SALT_AR1 = 0x41523120
EPS = 2.0 ** -52


def normals(B, n_obs, seed, offset=0):
    """(z, rad) of shape (B, n_obs): z[:, k] as ar1.cu draws it and its Box-Muller radius."""
    nb = (n_obs + 1) // 2
    rows = streams.rows_of(B, offset)[:, None]
    m = np.arange(nb, dtype=np.uint64)[None, :]
    n0, n1, rad = streams.normal2(streams._block(rows, m, SALT_AR1, seed))
    z = np.empty((B, 2 * nb))
    r = np.empty((B, 2 * nb))
    z[:, 0::2], z[:, 1::2] = n0, n1
    r[:, 0::2], r[:, 1::2] = rad, rad
    return z[:, :n_obs], r[:, :n_obs]


def sim_ar1(phi, n_obs, seed, offset=0):
    """(X (B, n_obs), err (B, n_obs)): the kernel's recursion on the replayed normals and a bound
    of the replay's error per element, for |phi| <= 1."""
    phi = np.asarray(phi, dtype=np.float64).reshape(-1)
    B = phi.shape[0]
    z, rad = normals(B, n_obs, seed, offset)
    dz = 1e-14 * np.maximum(1.0, rad)
    X = np.empty((B, n_obs))
    err = np.empty((B, n_obs))
    x, dx = np.zeros(B), np.zeros(B)
    for t in range(n_obs):
        x_new = phi * x + z[:, t]
        # the innovation's error, the previous error through phi, the two roundings of the step
        dx = np.abs(phi) * dx + dz[:, t] + 2 * EPS * (np.abs(phi * x) + np.abs(x_new))
        x = x_new
        X[:, t] = x
        err[:, t] = 4 * dx
    return X, err
