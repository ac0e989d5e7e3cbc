"""CPU test double of the stochastic volatility entry point -- TEST INFRASTRUCTURE ONLY.

Extends tests/abi_double.py and tests/priors_double.py (TABLE goes after theirs) with a
restatement, on host pointers, of elfi_b200_sim_svm_f64: the reference's arithmetic (SciPy's
levy_stable formula in S0 and the AR(1) log-volatility) on uniforms and normals from a NumPy
RandomState instead of the device's Philox streams (same distribution, deterministic in
(seed, offset)), and the kurt / skew of np.quantile.  elfi_b200_row_quantiles_f64 comes from
tests/mg1_double.py.
"""
import numpy as np

import abi_double as d
import mg1_double
import svm_replay
from elfi_b200 import ops


def svm_data(P, n, rs):
    """(B, n) data of parameters P (B, 7); NaN rows where the reference raises."""
    B = P.shape[0]
    u_th, u_w = 1.0 - rs.random_sample((B, n)), 1.0 - rs.random_sample((B, n))
    z = rs.standard_normal((B, n))
    v, _, _ = svm_replay.stable(*(P[:, k:k + 1] for k in range(4)), u_th, u_w)
    x, _, scale0 = svm_replay.log_vol(P, z, np.ones((B, n)))
    with np.errstate(all='ignore'):
        y = np.exp(0.5 * x) * v
    y[~svm_replay.params_ok(P, scale0)] = np.nan
    return y


def summaries(y):
    with np.errstate(all='ignore'):
        q = np.quantile(y, ops.SVM_LEVELS, axis=1)
        return np.column_stack([(q[4] - q[0]) / (q[3] - q[1]),
                                ((q[4] - q[2]) - (q[2] - q[0])) / (q[4] - q[0])])


def sim_svm_f64(ctx, P, ldP, B, n_obs, seed, offset, Y, ldY, S, ldS, stream):
    d._require(ldP >= 7 and ops.MG1_NOBS_MIN <= n_obs <= ops.MG1_NOBS_MAX, 'sim_svm: bad shape')
    d._require(not d._addr(S) or ldS >= 2, 'sim_svm: bad shape')
    if not B:
        return
    y = svm_data(np.array(d._mat(P, B, 7, ldP)), n_obs, d._rs(seed, offset, 43))
    if d._addr(Y):
        d._mat(Y, B, n_obs, ldY)[:] = y
    if d._addr(S):
        d._mat(S, B, 2, ldS)[:] = summaries(y)


TABLE = {'elfi_b200_sim_svm_f64': sim_svm_f64,
         'elfi_b200_row_quantiles_f64': mg1_double.row_quantiles_f64}
