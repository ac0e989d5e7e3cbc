"""NumPy restatement of the ROMC kernels of include/elfi_b200.h (elfi_b200_romc_*) and their CPU
test double -- TEST INFRASTRUCTURE ONLY.

The functions state each kernel's definition on host arrays: `nm_init` / `nm_step` the lock-step
Nelder-Mead state machine (scipy's _minimize_neldermead, one point per call, stable vertex order
with NaN last), `ls_init` / `ls_step` the line search, `box_sample` the Philox box draws,
`weights` and `posterior_unnorm`.  `TABLE` routes the entry points here on top of
tests/abi_double.py (through `abi_double.install`), so the unmodified ROMC host code
runs without a GPU.
"""
import numpy as np

import abi_double as d
import streams

INIT, REFLECT, EXPAND, CONTRACT_OUT, CONTRACT_IN, SHRINK, DONE = range(7)
NM_INTS = 8
SALT = 0x524f4d43


def nm_doubles(p):
    return (p + 1) * (p + 1) + 3 * p + 2


def _stable_order(f):
    key = np.where(np.isnan(f), 1, 0)
    return np.lexsort((np.arange(len(f)), np.where(np.isnan(f), 0.0, f), key))


def nm_init(x0):
    """State (P, nm_doubles(p)), int state (P, 8) and the first points (P, p)."""
    x0 = np.asarray(x0, dtype=np.float64)
    P, N = x0.shape
    st = np.zeros((P, nm_doubles(N)))
    ist = np.zeros((P, NM_INTS), dtype=np.int32)
    for i in range(P):
        sim = np.empty((N + 1, N))
        sim[0] = x0[i]
        for k in range(N):
            y = x0[i].copy()
            y[k] = (1 + 0.05) * y[k] if y[k] != 0 else 0.00025
            sim[k + 1] = y
        st[i, :(N + 1) * N] = sim.ravel()
        st[i, (N + 1) * N:(N + 1) * (N + 1)] = np.inf
        ist[i, :5] = [INIT, 0, 1, 0, -1]
    return st, ist, x0.copy()


def nm_step(st, ist, f, theta, maxiter, maxfev, xatol=1e-4, fatol=1e-4):
    """One call of elfi_b200_romc_nm_step_f64 on host arrays (updated in place)."""
    P, N = theta.shape
    for i in range(P):
        if ist[i, 0] == DONE:
            continue
        _nm_one(st[i], ist[i], float(f[i]), theta[i], N, maxiter, maxfev, xatol, fatol)


def _nm_one(s, st, f, out, N, maxiter, maxfev, xatol, fatol):
    sim = s[:(N + 1) * N].reshape(N + 1, N)
    o = (N + 1) * N
    fsim = s[o:o + N + 1]
    xbar, xr, xt = s[o + N + 1:o + 2 * N + 1], s[o + 2 * N + 1:o + 3 * N + 1], \
        s[o + 3 * N + 1:o + 4 * N + 1]
    phase, nit, nfev, j = (int(v) for v in st[:4])
    propose, end, counted, top = None, False, False, False
    if phase == INIT:
        fsim[j] = f
        j += 1
        if j <= N and nfev < maxfev:
            propose = sim[j]
        else:
            nit, end, counted = 0, True, True
    elif phase == REFLECT:
        s[-2] = f
        if f < fsim[0]:
            xt[:] = 3.0 * xbar - 2.0 * sim[-1]
            phase = EXPAND
        elif f < fsim[-2]:
            sim[-1], fsim[-1] = xr, f
            end = counted = True
        elif f < fsim[-1]:
            xt[:] = 1.5 * xbar - 0.5 * sim[-1]
            phase = CONTRACT_OUT
        else:
            xt[:] = 0.5 * xbar + 0.5 * sim[-1]
            phase = CONTRACT_IN
        if not end:
            if nfev < maxfev:
                propose = xt
            else:
                end = True
    elif phase == EXPAND:
        if f < s[-2]:
            sim[-1], fsim[-1] = xt, f
        else:
            sim[-1], fsim[-1] = xr, s[-2]
        end = counted = True
    if phase in (CONTRACT_OUT, CONTRACT_IN, SHRINK) and not end and propose is None:
        shrink = True
        if phase != SHRINK:
            if (f <= s[-2]) if phase == CONTRACT_OUT else (f < fsim[-1]):
                sim[-1], fsim[-1] = xt, f
                end = counted = True
                shrink = False
            else:
                j = 0
        else:
            fsim[j] = f
        if shrink:
            phase = SHRINK
            j += 1
            if j > N:
                end = counted = True
            else:
                sim[j] = sim[0] + 0.5 * (sim[j] - sim[0])
                if nfev < maxfev:
                    propose = sim[j]
                else:
                    end = True
    if end:
        if counted:
            nit += 1
        ind = _stable_order(fsim)
        sim[:] = sim[ind]
        fsim[:] = fsim[ind]
        top = True
    if top:
        finish = not (nfev < maxfev and nit < maxiter)
        if not finish:
            finish = bool(np.max(np.abs(sim[1:] - sim[0])) <= xatol and
                          np.max(np.abs(fsim[0] - fsim[1:])) <= fatol)
        if finish:
            s[-1] = np.min(fsim)
            st[4] = 1 if nfev >= maxfev else (2 if nit >= maxiter else 0)
            phase = DONE
            out[:] = sim[0]
        else:
            xbar[:] = np.add.reduce(sim[:-1], 0) / N
            xr[:] = 2.0 * xbar - sim[-1]
            phase = REFLECT
            propose = xr
    if propose is not None:
        out[:] = propose
        nfev += 1
    st[:4] = [phase, nit, nfev, j]


def ls_init(x_min, active):
    P, N = x_min.shape
    st = np.zeros((2 * N * P, N + 2))
    ist = np.zeros((2 * N * P, 4), dtype=np.int32)
    for t in range(2 * N * P):
        st[t, :N] = x_min[t % P]
        ist[t, 2] = 0 if active[t % P] else 1
    return st, ist, np.tile(x_min, (2 * N, 1, 1))


def ls_step(st, ist, f, theta, rot, eps, K, eta0, rep_lim, limits):
    """One call of elfi_b200_romc_line_search_f64 (init = 0) on host arrays; eta0 only seeds the
    state at init, so the state's eta is used here."""
    n2p, P, N = theta.shape
    f = np.asarray(f).reshape(n2p, P)
    for dp in range(n2p):
        d, side = dp >> 1, dp & 1
        for i in range(P):
            t = dp * P + i
            if ist[t, 2]:
                continue
            th, offset, eta = st[t, :N], st[t, N], st[t, N + 1]
            k, rep = int(ist[t, 0]), int(ist[t, 1])
            vd = rot[i][:, d] if side else -rot[i][:, d]
            done = False
            if f[dp, i] < eps and rep <= rep_lim:
                th += eta * vd
                offset += eta
                rep += 1
            else:
                th -= eta * vd
                offset -= eta
                if rep > rep_lim:
                    done = True
                else:
                    eta = eta / 2
                    k += 1
                    rep = 0
                    done = k >= K
            if done:
                if offset <= 0:
                    offset = eta
                limits[i, d, side] = offset if side else -offset
                ist[t, 2] = 1
            st[t, N], st[t, N + 1] = offset, eta
            ist[t, 0], ist[t, 1] = k, rep
            theta[dp, i] = th


def _uniforms(seed, r, j, N):
    u = np.empty(N)
    for dd in range(0, N, 2):
        w = streams.philox4x32_10(np.uint32(j), np.uint32(r), np.uint32(dd >> 1), np.uint32(SALT),
                                  seed)
        w = [int(np.asarray(v).reshape(-1)[0]) for v in w]
        u[dd] = streams.u01(w[0], w[1])
        if dd + 1 < N:
            u[dd + 1] = streams.u01(w[2], w[3])
    return u


def contains(x, rinv, c, lim):
    """NDimBoundingBox.contains with the products summed in order."""
    N = len(x)
    for r in range(N):
        a = b = 0.0
        for k in range(N):
            a += rinv[r, k] * x[k]
            b += rinv[r, k] * -c[k]
        y = a + b
        if y < lim[r, 0] or y > lim[r, 1]:
            return False
    return True


def quad(x, coef):
    s = coef[0]
    e = 1
    N = len(x)
    for a in range(N):
        s += coef[e] * x[a]
        e += 1
    for a in range(N):
        for b in range(a, N):
            s += coef[e] * (x[a] * x[b])
            e += 1
    return s


def box_sample(center, rot, rot_inv, limits, volume, n2, seed, coef=None):
    R, N = center.shape
    pts = np.empty((R, n2, N))
    q = np.empty((R, n2))
    surr = None if coef is None else np.empty((R, n2))
    for r in range(R):
        for j in range(n2):
            u = _uniforms(seed, r, j, N)
            t = limits[r, :, 0] + (limits[r, :, 1] - limits[r, :, 0]) * u
            x = np.array([sum_in_order(rot[r, a] * t) for a in range(N)]) + center[r]
            pts[r, j] = x
            q[r, j] = 1.0 / volume[r] if contains(x, rot_inv[r], center[r], limits[r]) else 0.0
            if surr is not None:
                surr[r, j] = quad(x, coef[r])
    return pts, q, surr


def sum_in_order(v):
    s = 0.0
    for e in v:
        s += e
    return s


def weights(dist, prior, q, eps):
    dist, prior, q = (np.asarray(a, dtype=np.float64) for a in (dist, prior, q))
    with np.errstate(invalid='ignore', divide='ignore'):
        return np.where(q > 0, (dist < eps) * prior / np.where(q > 0, q, 1.0), 0.0)


def posterior_unnorm(theta, prior, eps, center=None, rot_inv=None, limits=None, coef=None,
                     fvals=None):
    theta = np.asarray(theta, dtype=np.float64)
    out = np.empty(len(theta))
    for m in range(len(theta)):
        if fvals is not None:
            count = int(np.sum(fvals[m] <= eps))
        else:
            count = sum(1 for k in range(len(center))
                        if contains(theta[m], rot_inv[k], center[k], limits[k]) and
                        quad(theta[m], coef[k]) <= eps)
        out[m] = prior[m] * count
    return out


# ---- the C ABI on host pointers --------------------------------------------------------------
def nm_init_f64(ctx, P, p, x0, ld_x0, state, istate, theta, ld_theta, stream):
    d._require(1 <= p <= 16, 'romc_nm_init: bad p')
    st, ist, th = nm_init(np.array(d._mat(x0, P, p, ld_x0)))
    d._mat(state, P, nm_doubles(p))[:] = st
    d._mat(istate, P, NM_INTS, dtype=np.int32)[:] = ist
    d._mat(theta, P, p, ld_theta)[:] = th


def nm_step_f64(ctx, P, p, state, istate, fvals, theta, ld_theta, maxiter, maxfev, xatol, fatol,
                stream):
    nm_step(d._mat(state, P, nm_doubles(p)), d._mat(istate, P, NM_INTS, dtype=np.int32),
            d._vec(fvals, P), d._mat(theta, P, p, ld_theta), maxiter, maxfev, xatol, fatol)


def line_search_f64(ctx, init, P, p, x_min, rot, active, state, istate, fvals, theta, eps, K, eta,
                    rep_lim, limits, stream):
    st = d._mat(state, 2 * p * P, p + 2)
    ist = d._mat(istate, 2 * p * P, 4, dtype=np.int32)
    th = d._mat(theta, 2 * p * P, p).reshape(2 * p, P, p)
    xm = np.array(d._mat(x_min, P, p))
    if init:
        s0, i0, t0 = ls_init(xm, np.array(d._vec(active, P, dtype=np.int32)))
        s0[:, p + 1] = eta
        st[:], ist[:], th[:] = s0, i0, t0
        return
    R = np.array(d._mat(rot, P, p * p)).reshape(P, p, p)
    lim = d._mat(limits, P, 2 * p).reshape(P, p, 2)
    ls_step(st, ist, np.array(d._mat(fvals, 2 * p, P)), th, R, eps, K, eta, rep_lim, lim)


def box_sample_f64(ctx, R, p, n2, center, rot, rot_inv, limits, volume, seed, coef, pts, q, surr,
                   stream):
    nc = 1 + p + p * (p + 1) // 2
    args = [np.array(d._mat(a, R, w)) for a, w in ((center, p), (rot, p * p), (rot_inv, p * p),
                                                   (limits, 2 * p))]
    cf = np.array(d._mat(coef, R, nc)) if d._addr(surr) else None
    P_, Q_, S_ = box_sample(args[0], args[1].reshape(R, p, p), args[2].reshape(R, p, p),
                            args[3].reshape(R, p, 2), np.array(d._vec(volume, R)), n2, seed, cf)
    d._mat(pts, R * n2, p)[:] = P_.reshape(-1, p)
    d._mat(q, R, n2)[:] = Q_
    if cf is not None:
        d._mat(surr, R, n2)[:] = S_


def weights_f64(ctx, n, dist, prior, q, eps, w, stream):
    d._vec(w, n)[:] = weights(d._vec(dist, n), d._vec(prior, n), d._vec(q, n), eps)


def posterior_unnorm_f64(ctx, M, R, p, theta, ld_theta, center, rot_inv, limits, coef, fvals, ld_f,
                         eps, prior, out, stream):
    nc = 1 + p + p * (p + 1) // 2
    th = np.array(d._mat(theta, M, p, ld_theta))
    pr = np.array(d._vec(prior, M))
    if d._addr(fvals):
        res = posterior_unnorm(th, pr, eps, fvals=np.array(d._mat(fvals, M, R, ld_f)))
    else:
        res = posterior_unnorm(th, pr, eps, np.array(d._mat(center, R, p)),
                               np.array(d._mat(rot_inv, R, p * p)).reshape(R, p, p),
                               np.array(d._mat(limits, R, 2 * p)).reshape(R, p, 2),
                               np.array(d._mat(coef, R, nc)))
    d._vec(out, M)[:] = res


TABLE = {'elfi_b200_romc_nm_init_f64': nm_init_f64,
         'elfi_b200_romc_nm_step_f64': nm_step_f64,
         'elfi_b200_romc_line_search_f64': line_search_f64,
         'elfi_b200_romc_box_sample_f64': box_sample_f64,
         'elfi_b200_romc_weights_f64': weights_f64,
         'elfi_b200_romc_posterior_unnorm_f64': posterior_unnorm_f64}
