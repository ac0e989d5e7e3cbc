"""NumPy replay of the Lorenz simulator's stream and step (elfi_b200/csrc/lorenz.cu) -- TEST
INFRASTRUCTURE ONLY.

Built on oracle/streams.py (the Philox generator, u01 and Box-Muller).  The normal of step s and
variable k of a row is Box-Muller normal (k & 1) of the block (row, row >> 32, (s << 6) | (k >> 1),
SALT_LORENZ); the replayed normals are within 1e-14 max(1, rad) of the device's (rad the Box-Muller
radius).  The RK4 step is the reference's NumPy code (examples.lorenz.runge_kutta_ode_solver), which
rounds every operation as the kernel does, so given the kernel's own y_{s-1} and the same eta a step
is bit-exact; the only difference comes from the normals' ulps, carried through eta.
"""
import numpy as np

import streams

SALT_LORENZ = 0x4C4F525A
EPS = 2.0 ** -52


def normals(B, T, m, seed, offset=0):
    """e (B, T - 1, m): the normal of steps s = 1 .. T - 1, and a bound of its replay error."""
    rows = streams.rows_of(B, offset)[:, None, None]
    s = np.arange(1, T, dtype=np.uint64)[None, :, None]
    k = np.arange(m, dtype=np.uint64)[None, None, :]
    blk = (s << np.uint64(6)) | (k >> np.uint64(1))
    n0, n1, rad = streams.normal2(streams._block(rows, blk, SALT_LORENZ, seed))
    e = np.where((k & np.uint64(1)) == 0, n0, n1)
    return e, 1e-14 * np.maximum(1.0, rad)


def eta_replay(e, err, phi, s_phi):
    """eta (B, T - 1, m) of every step from the normals, and a bound of its error."""
    eta = np.zeros(e.shape)
    bound = np.zeros(e.shape)
    cur = np.zeros(e.shape[::2])
    cb = np.zeros(e.shape[::2])
    for s in range(e.shape[1]):
        cur = phi * cur + e[:, s] * s_phi
        cb = abs(phi) * cb + abs(s_phi) * err[:, s] + 2 * EPS * np.abs(cur)
        eta[:, s], bound[:, s] = cur, cb
    return eta, bound


def rk4_step(y, eta, theta1, theta2, f, dt):
    """One step of every row from y (B, m) with forcing eta (B, m)."""
    from elfi_b200.examples import lorenz
    return lorenz.runge_kutta_ode_solver(lorenz._lorenz_ode, dt, y,
                                         (eta, theta1.reshape(-1, 1), theta2.reshape(-1, 1), f))


def one_step_bound(y_new, eta_bound, dt):
    """|y_s(device) - y_s(replay)| bound from eta's error: dy / d eta_j is dt (own variable) plus
    O(dt^2) couplings to the neighbours, and a few ulp of rounding that the difference may flip."""
    e = eta_bound.max(axis=1, keepdims=True)
    return 4.0 * dt * e + 16 * EPS * (np.abs(y_new) + 1.0)
