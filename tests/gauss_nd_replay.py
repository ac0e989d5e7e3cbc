"""NumPy replay of the n-D Gaussian mean streams (elfi_b200/csrc/gauss_nd.cu) -- TEST INFRASTRUCTURE
ONLY.

Built on oracle/streams.py (the Philox generator, u01 and Box-Muller): the normals of a row are
numbered q = t D + k, and block q // 2 gives normals 2 (q // 2) and 2 (q // 2) + 1.  The replayed
normals are within 1e-14 max(1, rad) of the device's (streams.py), and the kernel's FMAs round once
where the replay rounds twice, so every element is compared within a bound carried from the normals'
error through the factor A, plus the roundings of the D - 1 additions and of the mean.
"""
import numpy as np

import streams

SALT_GAUSS_ND = 0x47534E44
EPS = 2.0 ** -52


def normals(B, n_obs, D, seed, offset=0):
    """(z, rad) of shape (B, n_obs, D): z[:, t, k] as gauss_nd.cu draws it, and its Box-Muller
    radius."""
    nq = n_obs * D
    nb = (nq + 1) // 2
    rows = streams.rows_of(B, offset)[:, None]
    m = np.arange(nb, dtype=np.uint64)[None, :]
    n0, n1, rad = streams.normal2(streams._block(rows, m, SALT_GAUSS_ND, seed))
    z = np.empty((B, 2 * nb))
    r = np.empty((B, 2 * nb))
    z[:, 0::2], z[:, 1::2] = n0, n1
    r[:, 0::2], r[:, 1::2] = rad, rad
    return z[:, :nq].reshape(B, n_obs, D), r[:, :nq].reshape(B, n_obs, D)


def sim_gauss_nd(mu, A, n_obs, seed, offset=0):
    """(Y (B, n_obs, D), err (B, n_obs, D)): y[t, j] = (sum_k z[t, k] A[k, j], k ascending) + mu_j
    on the replayed normals, and a bound of the replay's error per element."""
    mu = np.asarray(mu, dtype=np.float64)
    A = np.asarray(A, dtype=np.float64)
    B, D = mu.shape
    z, rad = normals(B, n_obs, D, seed, offset)
    dz = 1e-14 * np.maximum(1.0, rad)
    s = z[:, :, 0, None] * A[0][None, None, :]
    mag = np.abs(s)
    err = np.abs(A[0])[None, None, :] * dz[:, :, 0, None]
    for k in range(1, D):
        term = z[:, :, k, None] * A[k][None, None, :]
        s = s + term
        mag = mag + np.abs(term)
        err = err + np.abs(A[k])[None, None, :] * dz[:, :, k, None]
    Y = s + mu[:, None, :]
    bound = 4 * (err + 2 * (D + 1) * EPS * (mag + np.abs(mu)[:, None, :] + np.abs(Y)))
    return Y, bound
