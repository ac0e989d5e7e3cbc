"""NumPy replay of the stochastic volatility streams (elfi_b200/csrc/svm.cu) -- TEST INFRASTRUCTURE
ONLY.

Built on oracle/streams.py (the Philox generator, u01 and Box-Muller): block j of (row, SALT_SVM)
gives TH = (1 - u01(x, y)) pi - pi / 2 and W = -log(u01(z, w)) of observation j, block m of
(row, SALT_SVM_N) the log-volatility normals z_{2m}, z_{2m+1}.  The uniforms are exact.  The shock is
SciPy's levy_stable formula (stable) in NumPy; it differs from the device's only through the ulps
of sin, cos, tan, arctan, pow and log, which `stable` carries through the formula to a bound
(extending toad_replay.step_bound to beta != 0 and the S0 shift).  The log-volatility is within a
bound carried through the AR(1) recurrence from the normals' error (as arch_replay does).
"""
import numpy as np

import streams

SALT_SVM = 0x53564D31
SALT_SVM_N = 0x53564D4E
EPS = 2.0 ** -52
R = 4 * EPS          # relative error allowed to each transcendental, CUDA's against NumPy's


def draws(B, n, seed, offset=0):
    """(u_th, u_w, z, rad), each (B, n): the angle and exponential uniforms of every shock, and the
    log-volatility normals with their Box-Muller radii."""
    rows = streams.rows_of(B, offset)[:, None]
    j = np.arange(n, dtype=np.uint64)[None, :]
    w = streams._block(rows, j, SALT_SVM, seed)
    u_th, u_w = 1.0 - streams.u01(w[0], w[1]), streams.u01(w[2], w[3])
    nb = (n + 1) // 2
    m = np.arange(nb, dtype=np.uint64)[None, :]
    n0, n1, rad = streams.normal2(streams._block(rows, m, SALT_SVM_N, seed))
    z = np.empty((B, 2 * nb))
    r = np.empty((B, 2 * nb))
    z[:, 0::2], z[:, 1::2] = n0, n1
    r[:, 0::2], r[:, 1::2] = rad, rad
    return u_th, u_w, z[:, :n], r[:, :n]


def stable(alpha, beta, kappa, eta, u_th, u_w, s0=True):
    """levy_stable(alpha, beta, loc=eta, scale=kappa).rvs from the uniforms, in SciPy's order
    (_rvs_Z1, vals * scale + loc, the S1 shift at alpha == 1, the S0 shift); arguments broadcast.

    Returns (x, err, cond): err bounds |device - x| where every transcendental may differ by R
    (relative) and every other operation is the same correctly rounded one, carried through the
    formula with absolute errors, so the cancellation of each sum is accounted for: the
    denominator cos TH / tan(alpha (th0 + TH)) + sin TH, the three-term numerator, the sum
    th0 + TH inside tan (whose relative slope is 2 / |sin 2y|) and the S0 subtraction.  cond is the
    largest condition number (|a| + |b|) / |a + b| of the denominator and numerator sums."""
    alpha, beta, kappa, eta, u_th, u_w = np.broadcast_arrays(
        *(np.asarray(a, dtype=np.float64) for a in (alpha, beta, kappa, eta, u_th, u_w)))
    with np.errstate(all='ignore'):
        TH = u_th * np.pi + (-np.pi / 2)
        W = -np.log(u_w) * 1.0 + 0.0
        eW = R * np.abs(W)
        aTH, bTH = alpha * TH, beta * TH
        cosTH, tanTH, sinTH = np.cos(TH), np.tan(TH), np.sin(TH)
        cos_a, sin_a = np.cos(aTH), np.sin(aTH)
        tan_a = np.tan(np.pi * alpha / 2)
        one, b0 = alpha == 1, beta == 0
        # alpha == 1
        h = np.pi / 2 + bTH
        arg = (np.pi / 2 * W * cosTH) / h
        lg = np.log(arg)
        e_lg = (2 * R + 3 * EPS) + R * np.abs(lg)           # log of an argument off by 2R + 3 EPS
        t_a, t_b = h * tanTH, beta * lg
        d1 = t_a - t_b
        e_d1 = np.abs(t_a) * (R + EPS) + np.abs(beta) * e_lg + EPS * (np.abs(t_b) + np.abs(d1))
        z_one = 2 / np.pi * d1
        e_one = 2 / np.pi * e_d1 + EPS * np.abs(z_one)
        # alpha != 1: beta == 0 takes th0 = 0, val0 = 0 (then the expressions are beta0func's)
        val0 = np.where(b0, 0.0, beta * tan_a)
        e_val0 = (R + EPS) * np.abs(val0)
        th0 = np.where(b0, 0.0, np.arctan(val0) / alpha)
        e_th0 = np.abs(th0) * (2 * R + 2 * EPS)              # arctan's condition number is <= 1
        s = np.where(b0, TH, th0 + TH)
        y = alpha * s
        e_y = alpha * (e_th0 + EPS * np.abs(s)) + EPS * np.abs(y)
        tan_y = np.where(b0, np.tan(aTH), np.tan(y))
        rel_tan = R + 2 * e_y / np.abs(np.sin(2 * y))
        t1 = cosTH / tan_y
        e_t1 = np.abs(t1) * (R + rel_tan + EPS)
        den = t1 + sinTH
        e_den = e_t1 + R * np.abs(sinTH) + EPS * np.abs(den)
        c_den = (np.abs(t1) + np.abs(sinTH)) / np.abs(den)
        A2 = sin_a * tanTH
        A = cos_a + A2
        e_A = R * np.abs(cos_a) + (2 * R + EPS) * np.abs(A2) + EPS * np.abs(A)
        B2 = cos_a * tanTH
        Bd = sin_a - B2
        e_B = R * np.abs(sin_a) + (2 * R + EPS) * np.abs(B2) + EPS * np.abs(Bd)
        C = val0 * Bd
        e_C = np.abs(val0) * e_B + e_val0 * np.abs(Bd) + EPS * np.abs(C)
        num = np.where(b0, A, A - C)
        e_num = np.where(b0, e_A, e_A + e_C + EPS * np.abs(num))
        c_num = np.where(b0, (np.abs(cos_a) + np.abs(A2)) / np.abs(A),
                         (np.abs(cos_a) + np.abs(A2) + np.abs(C)) / np.abs(num))
        val3 = W / den
        rel_val3 = R + e_den / np.abs(den) + EPS
        ratio = num / W
        rel_ratio = e_num / np.abs(num) + R + EPS
        pw = ratio ** (1.0 / alpha)
        rel_pw = rel_ratio / alpha + R
        z_not = val3 * pw
        e_not = np.abs(z_not) * (rel_val3 + rel_pw + EPS)
        Z1 = np.where(one, z_one, z_not)
        eZ = np.where(one, e_one, e_not)
        X = Z1 * kappa + eta
        eX = eZ * kappa + EPS * (np.abs(Z1 * kappa) + np.abs(X))
        shift1 = 2 * beta * kappa * np.log(kappa) / np.pi
        e_shift1 = np.abs(shift1) * (R + 4 * EPS)
        X1 = np.where(one, X + shift1, X)
        eX = np.where(one, eX + e_shift1 + EPS * np.abs(X1), eX)
        if s0:
            shift = np.where(one, beta * 2 * kappa * np.log(kappa) / np.pi,
                             kappa * beta * np.tan(np.pi * alpha / 2.0))
            out = X1 - shift
            eX = eX + np.abs(shift) * (R + 4 * EPS) + EPS * np.abs(out)
        else:
            out = X1
        cond = np.where(one, 1.0, np.maximum(c_den, c_num))
    return out, 2.0 * eX, cond


def log_vol(P, z, rad):
    """(x (B, n), err (B, n)): the kernel's AR(1) on the replayed normals and a bound of the
    replay's error (the normals within 1e-14 max(1, rad), streams.py, plus each step's roundings)."""
    mu, phi, sigma = (P[:, k:k + 1] for k in (4, 5, 6))
    with np.errstate(all='ignore'):
        scale0 = sigma / np.sqrt(1 - np.minimum(phi ** 2, 0.99999))
        dz = 1e-14 * np.maximum(1.0, rad)
        x = np.empty(z.shape)
        err = np.empty(z.shape)
        x[:, :1] = z[:, :1] * scale0 + mu
        err[:, :1] = scale0 * dz[:, :1] + 2 * EPS * (np.abs(z[:, :1] * scale0) + np.abs(x[:, :1]))
        for t in range(1, z.shape[1]):
            loc = mu + phi * (x[:, t - 1:t] - mu)
            x[:, t:t + 1] = z[:, t:t + 1] * sigma + loc
            err[:, t:t + 1] = np.abs(phi) * err[:, t - 1:t] + sigma * dz[:, t:t + 1] + 4 * EPS * (
                np.abs(x[:, t - 1:t]) + np.abs(mu) + np.abs(loc) + np.abs(z[:, t:t + 1] * sigma) +
                np.abs(x[:, t:t + 1]))
    return x, err, scale0[:, 0]


def params_ok(P, scale0):
    a, b, k, s = P[:, 0], P[:, 1], P[:, 2], P[:, 6]
    with np.errstate(invalid='ignore'):
        return (a > 0) & (a <= 2) & (b >= -1) & (b <= 1) & (k >= 0) & (s >= 0) & (scale0 >= 0)


def sim_svm(P, n, seed, offset=0):
    """(Y, err, v, v_err, x, cond), each (B, n) but cond: the kernel's data on the replayed draws and
    a bound of the replay's error per element; NaN rows where the reference raises."""
    P = np.asarray(P, dtype=np.float64)
    u_th, u_w, z, rad = draws(P.shape[0], n, seed, offset)
    cols = [P[:, k:k + 1] for k in range(4)]
    v, v_err, cond = stable(*cols, u_th, u_w)
    x, x_err, scale0 = log_vol(P, z, rad)
    with np.errstate(all='ignore'):
        e = np.exp(0.5 * x)
        Y = e * v
        err = e * v_err + np.abs(Y) * (0.5 * x_err * 1.01 + R + 2 * EPS)
    bad = ~params_ok(P, scale0)
    Y[bad] = np.nan
    return Y, err, v, v_err, x, cond
