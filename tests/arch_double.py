"""CPU test double of the ARCH(1) entry points -- TEST INFRASTRUCTURE ONLY.

Extends tests/abi_double.py (through `abi_double.install`) with restatements of
elfi_b200_sim_arch_f64 and elfi_b200_arch_summaries_f64 on host pointers.  The summaries are the
reference's NumPy code (elfi_b200.examples.arch on host arrays); the simulator runs the reference's
recurrence on normals from a NumPy RandomState instead of the device's Philox streams (same
distribution, deterministic in (seed, offset)), and the fused summaries are those of exactly the
data the unfused form writes, as on the device.
"""
from itertools import combinations

import numpy as np

import abi_double as d
from elfi_b200 import ops


def summaries(x, n_lags):
    from elfi_b200.examples import arch
    with np.errstate(all='ignore'):
        cols = [arch.sample_mean(x), arch.sample_variance(x)]
        cols += [arch.autocorr(x, i) for i in range(1, n_lags + 1)]
        cols += [arch.pairwise_autocorr(x, i, j) for i, j in combinations(range(1, n_lags + 1), 2)]
    return np.column_stack(cols)


def arch_data(P, n_obs, rs):
    """The reference's recurrence (arch.py:100-132) on z (B, n_obs + 1): z[:, 0] = e_0, z[:, k] =
    xi_k, the normals of the device's layout."""
    z = rs.randn(P.shape[0], n_obs + 1)
    y = np.zeros((P.shape[0], n_obs + 1))
    e = z[:, 0]
    with np.errstate(all='ignore'):
        for k in range(1, n_obs + 1):
            e = z[:, k] * np.sqrt(0.2 + P[:, 1] * np.power(e, 2))
            y[:, k] = P[:, 0] * y[:, k - 1] + e
    return y[:, 1:]


def _shape_ok(n, n_lags, ldS):
    return (ops.ARCH_NOBS_MIN <= n <= ops.ARCH_NOBS_MAX and 1 <= n_lags <= ops.ARCH_LAGS_MAX and
            n_lags < n and ldS >= ops.arch_nsumm(n_lags))


def sim_arch_f64(ctx, P, ldP, B, n_obs, n_lags, seed, offset, Y, ldY, S, ldS, stream):
    d._require(ldP >= 2 and _shape_ok(n_obs, n_lags, ldS if d._addr(S) else 10 ** 9),
               'sim_arch: bad shape')
    if not B:
        return
    y = arch_data(np.array(d._mat(P, B, 2, ldP)), n_obs, d._rs(seed, offset, 31))
    if d._addr(Y):
        d._mat(Y, B, n_obs, ldY)[:] = y
    if d._addr(S):
        d._mat(S, B, ops.arch_nsumm(n_lags), ldS)[:] = summaries(y, n_lags)


def arch_summaries_f64(ctx, X, ld_b, ld_j, B, n, n_lags, S, ldS, stream):
    d._require(_shape_ok(n, n_lags, ldS), 'arch_summaries: bad shape')
    if not B:
        return
    span = (B - 1) * ld_b + (n - 1) * ld_j + 1
    x = np.array(np.lib.stride_tricks.as_strided(d._vec(X, span), (B, n), (8 * ld_b, 8 * ld_j)))
    d._mat(S, B, ops.arch_nsumm(n_lags), ldS)[:] = summaries(x, n_lags)


TABLE = {'elfi_b200_' + f.__name__: f for f in (sim_arch_f64, arch_summaries_f64)}
