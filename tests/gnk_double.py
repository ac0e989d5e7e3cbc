"""CPU test double of the g-and-k summary entry points -- TEST INFRASTRUCTURE ONLY.

Extends tests/abi_double.py (through `abi_double.install`) with restatements of
elfi_b200_gnk_summaries_f64, elfi_b200_sim_gnk_summaries_f64, elfi_b200_sim_bignk_f64 and
elfi_b200_euclidean_multiss_f64 on host pointers.  The summaries are the reference's NumPy code
(elfi_b200.examples.gnk on host arrays); the simulators draw from a NumPy RandomState instead of
the device's Philox streams (same distributions, deterministic in (seed, offset)), and the fused
forms summarise exactly the data the unfused forms write, as on the device.
"""
import ctypes

import numpy as np

import abi_double as d
from elfi_b200 import ops

KINDS = {v: k for k, v in ops.GNK_KINDS.items()}


def _series(p, B, n, dim, ld_row, ld_obs):
    if B == 0:
        return np.empty((0, n, dim))
    nbytes = ((B - 1) * ld_row + (n - 1) * ld_obs + dim) * 8
    flat = np.frombuffer((ctypes.c_char * nbytes).from_address(d._addr(p)), dtype=np.float64)
    return np.lib.stride_tricks.as_strided(flat, (B, n, dim), (ld_row * 8, ld_obs * 8, 8))


def _summarise(y, kind):
    from elfi_b200.examples import gnk
    d._require(kind in KINDS, 'unknown kind {}'.format(kind))
    with np.errstate(invalid='ignore'):
        fn = gnk.ss_robust if KINDS[kind] == 'ss_robust' else gnk.ss_octile
        return fn(np.ascontiguousarray(y))[:, :, 0]


def _check_picks(picks_host, n):
    p = d._vec(picks_host, 21)
    d._require(p is not None and np.array_equal(p, ops.gnk_picks(n)), 'picks do not match n')


def gnk_summaries_f64(ctx, X, ld_row, ld_obs, B, n, dim, kind, picks_host, out, ld_out, stream):
    d._require(1 <= n <= ops.GNK_SERIES_MAX and dim in (1, 2), 'gnk_summaries: bad shape')
    _check_picks(picks_host, n)
    if B:
        s = _summarise(_series(X, B, n, dim, ld_row, ld_obs), kind)
        d._mat(out, B, s.shape[1], ld_out)[:] = s


def _gnk_data(A, Bs, g, k, c, B, n_obs, seed, offset):
    Y = np.empty((B, n_obs))
    d.sim_gnk_f64(None, A, Bs, g, k, c, B, n_obs, seed, offset, ctypes.c_void_p(Y.ctypes.data),
                  n_obs, None)
    return Y


def sim_gnk_summaries_f64(ctx, A, Bs, g, k, c, B, n_obs, seed, offset, kind, picks_host, out, ld_out,
                          stream):
    d._require(1 <= n_obs <= ops.GNK_FUSED_MAX, 'sim_gnk_summaries: bad shape')
    _check_picks(picks_host, n_obs)
    if B:
        s = _summarise(_gnk_data(A, Bs, g, k, c, B, n_obs, seed, offset)[:, :, None], kind)
        d._mat(out, B, s.shape[1], ld_out)[:] = s


def bignk_data(P, c, n_obs, rs):
    """The device's formula on NumPy normals: z1 = n0, z2 = rho n0 + sqrt(1 - rho^2) n1."""
    from streams import gnk_quantile
    n0, n1 = rs.randn(len(P), n_obs), rs.randn(len(P), n_obs)
    rho = P[:, 8:9]
    with np.errstate(invalid='ignore'):
        z1 = np.where(np.abs(rho) <= 1.0, n0, np.nan)
        z2 = rho * n0 + np.sqrt(1.0 - rho * rho) * n1
        return np.stack([gnk_quantile(P[:, 0:1], P[:, 2:3], P[:, 4:5], P[:, 6:7], c, z1),
                         gnk_quantile(P[:, 1:2], P[:, 3:4], P[:, 5:6], P[:, 7:8], c, z2)], axis=2)


def sim_bignk_f64(ctx, P, ldP, c, B, n_obs, seed, offset, Y, ldY, kind, picks_host, S, ldS, stream):
    d._require(n_obs >= 1 and ldP >= 9, 'sim_bignk: bad shape')
    if d._addr(S):
        d._require(n_obs <= ops.GNK_FUSED_MAX, 'sim_bignk: fused summaries need n_obs <= 512')
        _check_picks(picks_host, n_obs)
    if not B:
        return
    y = bignk_data(d._mat(P, B, 9, ldP), c, n_obs, d._rs(seed, offset, 9))
    if d._addr(Y):
        d._mat(Y, B, 2 * n_obs, ldY)[:] = y.reshape(B, 2 * n_obs)
    if d._addr(S):
        s = _summarise(y, kind)
        d._mat(S, B, s.shape[1], ldS)[:] = s


def euclidean_multiss_f64(ctx, S, ldS, B, K, obs, out, stream):
    from elfi_b200.examples import gnk
    d._require(1 <= K <= 128, 'euclidean_multiss: bad shape')
    if B:
        d._vec(out, B)[:] = gnk.euclidean_multiss(d._mat(S, B, K, ldS)[:, :, None],
                                                  observed=[d._vec(obs, K)[None, :, None]])


TABLE = {'elfi_b200_' + f.__name__: f for f in (
    gnk_summaries_f64, sim_gnk_summaries_f64, sim_bignk_f64, euclidean_multiss_f64)}
