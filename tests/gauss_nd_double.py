"""CPU test double of the n-D Gaussian mean entry points -- TEST INFRASTRUCTURE ONLY.

Extends tests/abi_double.py (through `abi_double.install`) with a NumPy statement of
elfi_b200_gauss_nd_summaries_f64, elfi_b200_gauss_nd_distance_f64 and elfi_b200_sim_gauss_nd_f64
on host pointers, in the orders the header states: every sum starts from 0.0; the sum over the
observations is NumPy's pairwise sum for D = 1 and a left fold for D >= 2; the distance's sum over
the D columns is a pairwise sum.  The simulator's data is tests/gauss_nd_replay.py (the kernel's
Philox streams, so the same rows as the device up to the last bits of the normals), and its
summaries are the statement's summaries of exactly that data, as on the device.
"""
import ctypes

import numpy as np

import abi_double as d
import gauss_nd_replay
from elfi_b200 import ops


def pairwise_sum(a):
    """NumPy's DOUBLE_pairwise_sum over the last axis of a (B, n) array, n >= 1: blocks of <= 128
    terms summed by 8 strided accumulators ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)) and a
    sequential tail; longer runs split at n / 2 rounded down to a multiple of 8."""
    n = a.shape[1]
    if n < 8:
        res = np.zeros(a.shape[0])
        for i in range(n):
            res = res + a[:, i]
        return res
    if n <= 128:
        r = [a[:, j].copy() for j in range(8)]
        i = 8
        while i < n - n % 8:
            r = [r[j] + a[:, i + j] for j in range(8)]
            i += 8
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        for k in range(i, n):
            res = res + a[:, k]
        return res
    n2 = n // 2
    n2 -= n2 % 8
    return pairwise_sum(a[:, :n2]) + pairwise_sum(a[:, n2:])


def axis1_sum(y):
    """np.sum(y, axis=1) of a C-contiguous (B, n, D) array in NumPy's order: from 0.0, a pairwise
    sum over n for D = 1 (the axis of length 1 is dropped), a left fold over t for D >= 2."""
    B, n, D = y.shape
    if D == 1:
        return (0.0 + pairwise_sum(y[:, :, 0]))[:, None]
    acc = np.zeros((B, D))
    for t in range(n):
        acc = acc + y[:, t, :]
    return acc


def meanvar(y):
    """(np.mean(y, axis=1), np.var(y, axis=1)) of (B, n, D) data in the orders of axis1_sum."""
    n = y.shape[1]
    with np.errstate(invalid='ignore', over='ignore'):
        mean = axis1_sum(y) / n
        c = y - mean[:, None, :]
        return mean, axis1_sum(c * c) / n


def distance(S, obs):
    """sqrt(np.sum((S - obs)**2., axis=1)) of (B, D) summaries: one pairwise sum per row."""
    with np.errstate(invalid='ignore', over='ignore'):
        c = S - obs[None, :]
        return np.sqrt(0.0 + pairwise_sum(c * c))


def _strided(p, B, n, D, ld_b, ld_t, ld_j):
    """(B, n, D) view with element strides (ld_b, ld_t, ld_j) over host memory."""
    last = (B - 1) * ld_b + (n - 1) * ld_t + (D - 1) * ld_j + 1
    buf = (ctypes.c_char * (8 * int(last))).from_address(d._addr(p))
    return np.lib.stride_tricks.as_strided(np.frombuffer(buf, dtype=np.float64), (B, n, D),
                                           (8 * ld_b, 8 * ld_t, 8 * ld_j))


def gauss_nd_summaries_f64(ctx, X, ld_b, ld_t, ld_j, B, n, D, out, ld_out, stream):
    d._require(B >= 0 and 1 <= n <= ops.GAUSS_ND_SUMM_NOBS_MAX and D >= 1 and ld_out >= 2 * D,
               'gauss_nd_summaries: bad shape')
    if not B:
        return
    mean, var = meanvar(np.ascontiguousarray(_strided(X, B, n, D, ld_b, ld_t, ld_j)))
    res = d._mat(out, B, 2 * D, ld_out)
    res[:, :D], res[:, D:] = mean, var


def gauss_nd_distance_f64(ctx, S, ld_b, ld_j, B, D, obs, d_out, stream):
    d._require(B >= 0 and 1 <= D <= ops.GAUSS_ND_SUMM_NOBS_MAX, 'gauss_nd_distance: bad shape')
    if not B:
        return
    Sm = np.ascontiguousarray(_strided(S, B, 1, D, ld_b, 0, ld_j)[:, 0, :])
    d._vec(d_out, B)[:] = distance(Sm, d._vec(obs, D).copy())


def sim_gauss_nd_f64(ctx, mu, ld_b, ld_j, B, D, A_host, n_obs, seed, offset, Y, ldY, S, ldS,
                     stream):
    d._require(0 <= B and 1 <= D <= ops.GAUSS_ND_D_MAX and 1 <= n_obs <= ops.GAUSS_ND_NOBS_MAX,
               'sim_gauss_nd: bad shape')
    d._require(d._addr(Y) or d._addr(S), 'sim_gauss_nd: nothing to produce')
    d._require((not d._addr(Y) or ldY >= n_obs * D) and (not d._addr(S) or ldS >= 2 * D),
               'sim_gauss_nd: bad leading dimension')
    if not B:
        return
    M = np.ascontiguousarray(_strided(mu, B, 1, D, ld_b, 0, ld_j)[:, 0, :])
    A = np.array(d._mat(A_host, D, D))
    y = gauss_nd_replay.sim_gauss_nd(M, A, n_obs, seed, offset)[0]
    if d._addr(Y):
        d._mat(Y, B, n_obs * D, ldY)[:] = y.reshape(B, -1)
    if d._addr(S):
        mean, var = meanvar(y)
        res = d._mat(S, B, 2 * D, ldS)
        res[:, :D], res[:, D:] = mean, var


TABLE = {'elfi_b200_' + f.__name__: f for f in (gauss_nd_summaries_f64, gauss_nd_distance_f64,
                                                 sim_gauss_nd_f64)}
