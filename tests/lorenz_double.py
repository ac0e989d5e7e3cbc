"""CPU test double of the Lorenz entry points -- TEST INFRASTRUCTURE ONLY.

Extends tests/abi_double.py (through `abi_double.install`) with restatements of
elfi_b200_sim_lorenz_f64 and elfi_b200_lorenz_summaries_f64 on host pointers.  The summaries are the
reference's NumPy code (elfi_b200.examples.lorenz on host arrays); the simulator is the reference's
recurrence on normals from a NumPy RandomState instead of the device's Philox streams (same
distribution, deterministic in (seed, offset)), with dt and sqrt(1 - phi^2) as passed, and the fused
summaries are those of exactly the data the unfused form writes, as on the device.
"""
import numpy as np

import abi_double as d
from elfi_b200 import ops


def lorenz_data(P, init, T, f, phi, s_phi, dt, rs):
    from elfi_b200.examples import lorenz
    B, m = P.shape[0], init.size
    X = np.empty((B, T, m))
    y = np.tile(init, (B, 1))
    X[:, 0] = y
    eta = np.zeros((B, m))
    th1, th2 = P[:, 0:1], P[:, 1:2]
    with np.errstate(all='ignore'):
        for s in range(1, T):
            eta = phi * eta + rs.standard_normal((B, m)) * s_phi
            y = lorenz.runge_kutta_ode_solver(lorenz._lorenz_ode, dt, y, (eta, th1, th2, f))
            X[:, s] = y
    return X


def _summaries(x):
    from elfi_b200.examples import lorenz
    with np.errstate(all='ignore'):
        return np.column_stack([lorenz.mean(x), lorenz.var(x), lorenz.autocov(x), lorenz.cov(x),
                                lorenz.xcov(x, True), lorenz.xcov(x, False)])


def sim_lorenz_f64(ctx, P, ldP, B, n_obs, n_timestep, init, f, phi, s_phi, dt, seed, offset, X, S,
                   ldS, stream):
    d._require(ops.LORENZ_NOBS_MIN <= n_obs <= ops.LORENZ_NOBS_MAX, 'sim_lorenz: bad n_obs')
    d._require(2 <= n_timestep <= ops.LORENZ_T_MAX and ldP >= 2, 'sim_lorenz: bad shape')
    if d._addr(S):
        d._require(ldS >= 6 and n_timestep * n_obs <= ops.LORENZ_SUMM_MAX_TERMS,
                   'sim_lorenz: summaries need n_timestep * n_obs <= 30728')
    if not B or not (d._addr(X) or d._addr(S)):
        return
    x = lorenz_data(d._mat(P, B, 2, ldP).copy(), d._vec(init, n_obs).copy(), n_timestep, f, phi,
                    s_phi, dt, d._rs(seed, offset, 13))
    if d._addr(X):
        d._mat(X, B, n_timestep * n_obs)[:] = x.reshape(B, -1)
    if d._addr(S):
        d._mat(S, B, 6, ldS)[:] = _summaries(x)


def lorenz_summaries_f64(ctx, X, ld_row, ld_t, ld_k, B, n_timestep, n_obs, S, ldS, stream):
    d._require(ops.LORENZ_SUMM_NOBS_MIN <= n_obs <= ops.LORENZ_NOBS_MAX and n_timestep >= 2 and
               n_timestep * n_obs <= ops.LORENZ_SUMM_MAX_TERMS, 'lorenz_summaries: bad shape')
    if not B:
        return
    span = (B - 1) * ld_row + (n_timestep - 1) * ld_t + (n_obs - 1) * ld_k + 1
    x = np.lib.stride_tricks.as_strided(d._vec(X, span), (B, n_timestep, n_obs),
                                        (8 * ld_row, 8 * ld_t, 8 * ld_k))
    d._mat(S, B, 6, ldS)[:] = _summaries(np.ascontiguousarray(x))


TABLE = {'elfi_b200_' + f.__name__: f for f in (sim_lorenz_f64, lorenz_summaries_f64)}
