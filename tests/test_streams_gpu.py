"""Throughput-mode generators element by element against the NumPy replay of their Philox
streams (oracle/streams.py).

The device draws are a deterministic function of (seed, row, block, salt), so every prior draw,
simulated observation and proposal is compared with an independent computation of the same value.
Tolerances are ulp-level, derived from the operations involved: the Philox words and u01 are exact,
the replayed Box-Muller normals are within 1e-14 max(1, rad) of the device's, and what follows
them (the MA2 recursion, mu + sigma z, the g-and-k quantile, mu + L z) propagates that bound.  A
stream-layout mistake (wrong counter word, two rows or pairs sharing a block, the wrong block for
z_2, z_3, a wrong bit mapping in u01) gives O(1) differences.  The statistical tests against the
reference's host path stay in tests/test_throughput_gpu.py: the reference draws from another RNG.
"""
import math

import numpy as np
import pytest
import scipy.stats as ss

import elfi_oracle as o
import streams

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -52


def _np(t):
    return t.cpu().numpy()


def _within(got, want, tol, what):
    bad = ~(np.abs(got - want) <= tol)
    assert not bad.any(), '{}: {} of {} differ, first at {}: {} vs {} (tol {})'.format(
        what, int(bad.sum()), bad.size, np.argwhere(bad)[0], got[bad][0], want[bad][0],
        np.broadcast_to(tol, bad.shape)[bad][0])


# ------------------------------------------------------------------------------ MA2 prior
@pytest.mark.parametrize('B,seed,offset', [(1, 3, 0), (255, 3, 0), (256, 3, 7), (257, 3, 0),
                                           (1000, 2 ** 32 + 5, 2 ** 32 - 500),
                                           (1000000, 0xDEADBEEF12345, 11)])
def test_prior_ma2_matches_replay(B, seed, offset):
    from elfi_b200 import ops
    t1, t2 = ops.prior_ma2(B, seed=seed, offset=offset)
    r1, r2 = streams.prior_ma2(B, seed, offset)
    _within(_np(t1), r1, 4 * EPS * 2.0, 't1')
    _within(_np(t2), r2, 4 * EPS * 3.0, 't2')
    only1 = ops.prior_ma2(B, seed=seed, offset=offset, which='t1')
    _within(_np(only1), r1, 4 * EPS * 2.0, 't1 alone')
    given = np.random.RandomState(B).uniform(-2, 2, B)
    cond = ops.prior_ma2(0, seed=seed, offset=offset, t1=given, which='t2')
    _within(_np(cond), streams.prior_ma2(B, seed, offset, mode=2, t1=given)[1], 4 * EPS * 3.0,
            't2 | t1')


# ------------------------------------------------------------------------------ MA2 simulator
def _ma2_params(rs, B):
    t1 = rs.uniform(-2, 2, B)
    t2 = rs.uniform(np.maximum(-1 - t1, -1 + t1), 1.0)
    corners = [(-2.0, 1.0), (2.0, 1.0), (0.0, -1.0), (1.999, 0.999), (-1.999, 0.999), (0.0, 1.0)]
    for j, (a, b) in enumerate(corners[:B]):
        t1[j], t2[j] = a, b
    return t1, t2


def _lag_tol(x, e, lag):
    """Bound of |autocov(X_device) - autocov(X_replay)| per row: 1e-12 of the mean |term| plus
    the propagated element bounds."""
    terms = np.abs(x[:, lag:] * x[:, :-lag])
    prop = np.abs(x[:, lag:]) * e[:, :-lag] + np.abs(x[:, :-lag]) * e[:, lag:]
    return 1e-12 * terms.mean(axis=1) + prop.mean(axis=1)


MA2_CASES = [(129, n) for n in (3, 4, 7, 8, 9, 15, 16, 17, 100, 129, 130, 257, 1000, 7688)] + \
            [(B, 100) for B in (1, 127, 128, 4097)] + [(4097, 130)]


@pytest.mark.parametrize('B,n_obs', MA2_CASES)
def test_sim_ma2_matches_replay(B, n_obs):
    from elfi_b200 import ops
    rs = np.random.RandomState(n_obs * 7 + B)
    t1, t2 = _ma2_params(rs, B)
    seed, offset = 2 ** 32 + 77, 2 ** 32 - 3
    Xr, err = streams.sim_ma2(t1, t2, n_obs, seed, offset)
    X, S = ops.sim_ma2(t1, t2, n_obs, seed=seed, offset=offset, want_data=True, want_summaries=True)
    X, S = _np(X), _np(S)
    _within(X, Xr, err, 'X')
    # the fused summaries are the autocovariances of the kernel's own X bit for bit ...
    assert np.array_equal(S[:, 0], o.autocov(X, 1)) and np.array_equal(S[:, 1], o.autocov(X, 2))
    # ... and within ulp-level bounds of those of the replayed data
    _within(S[:, 0], np.mean(Xr[:, 1:] * Xr[:, :-1], axis=1), _lag_tol(Xr, err, 1), 'S lag 1')
    _within(S[:, 1], np.mean(Xr[:, 2:] * Xr[:, :-2], axis=1), _lag_tol(Xr, err, 2), 'S lag 2')
    _, S_only = ops.sim_ma2(t1, t2, n_obs, seed=seed, offset=offset)
    assert np.array_equal(_np(S_only), S)
    X_only, none = ops.sim_ma2(t1, t2, n_obs, seed=seed, offset=offset, want_data=True,
                               want_summaries=False)
    assert none is None and np.array_equal(_np(X_only), X)


# ------------------------------------------------------------------------------ Gaussian model
@pytest.mark.parametrize('n_obs', [1, 2, 7, 8, 9, 128, 129, 7688])
def test_sim_gauss_matches_replay(n_obs):
    from elfi_b200 import ops
    rs = np.random.RandomState(n_obs)
    B = 257
    mu, sigma = rs.uniform(-1, 9, B), rs.uniform(0.01, 10, B)
    seed, offset = 2 ** 33 + 1, 2 ** 32 - 100
    Yr, err = streams.sim_gauss(mu, sigma, n_obs, seed, offset)
    Y, S = ops.sim_gauss(mu, sigma, n_obs, seed=seed, offset=offset, want_data=True)
    Y, S = _np(Y), _np(S)
    _within(Y, Yr, err, 'Y')
    assert np.array_equal(S[:, 0], np.mean(Y, axis=1)) and np.array_equal(S[:, 1], np.var(Y, axis=1))
    m = np.mean(Yr, axis=1)
    _within(S[:, 0], m, 1e-12 * np.mean(np.abs(Yr), axis=1) + err.mean(axis=1), 'mean')
    c = np.abs(Yr - m[:, None])
    e2 = 2 * err.max(axis=1)
    tol = 1e-12 * np.mean(c * c, axis=1) + 2 * np.mean(c, axis=1) * e2 + e2 ** 2
    _within(S[:, 1], np.var(Yr, axis=1), tol, 'var')
    _, S_only = ops.sim_gauss(mu, sigma, n_obs, seed=seed, offset=offset)
    assert np.array_equal(_np(S_only), S)


GAUSS_PRIORS = [(-1.0, 10.0, 0.01, 10.0), (0.0, 1.0, 3.0, 8.0), (0.0, 1.0, 6.0, 9.0),
                (0.0, 1.0, 9.0, 12.0), (2.0, 0.5, -12.0, -9.0)]


@pytest.mark.parametrize('prm', GAUSS_PRIORS)
def test_prior_gauss_matches_replay_and_truncnorm(prm):
    """Draws vs the replay, the KS test vs scipy.stats.truncnorm, and logprior_gauss vs
    truncnorm.logpdf -- also deep in either tail, where Phi(a) rounds to 1 unless the truncation
    is mirrored."""
    from elfi_b200 import ops
    mu_lo, mu_w, a, b = prm
    B, seed, offset = 100000, 2 ** 32 + 3, 5
    mu, sigma = ops.prior_gauss(B, seed=seed, prm=list(prm), offset=offset)
    mu, sigma = _np(mu), _np(sigma)
    rmu, rsigma = streams.prior_gauss(B, seed, prm, offset)
    _within(mu, rmu, 4 * EPS * (abs(mu_lo) + abs(mu_w)), 'mu')
    _within(sigma, rsigma, 1e-13 * np.abs(rsigma), 'sigma')
    assert np.all((sigma >= a) & (sigma <= b))
    assert np.unique(sigma).size > 0.99 * B
    assert ss.kstest(sigma, ss.truncnorm(a, b).cdf).pvalue > 1e-3
    assert ss.kstest(mu, ss.uniform(mu_lo, mu_w).cdf).pvalue > 1e-3
    rs = np.random.RandomState(1)
    theta = np.column_stack([rs.uniform(mu_lo - 0.1 * mu_w, mu_lo + 1.1 * mu_w, 4000),
                             rs.uniform(a - 0.1 * (b - a), b + 0.1 * (b - a), 4000)])
    theta[:4, 1] = [a, b, 0.5 * (a + b), np.nextafter(b, np.inf)]
    theta[:4, 0] = mu_lo + 0.5 * mu_w
    with np.errstate(divide='ignore'):
        ref = ss.uniform.logpdf(theta[:, 0], mu_lo, mu_w) + ss.truncnorm.logpdf(theta[:, 1], a, b)
    got = _np(ops.logprior_gauss(theta, list(prm)))
    assert np.array_equal(np.isfinite(got), np.isfinite(ref))
    fin = np.isfinite(ref)
    # rtol 1e-12 of the value, and 1e-13 of the terms it is the sum of (in a tail truncation
    # the log density crosses zero between terms of size 40)
    mass = streams.gauss_prior_constants(prm)[4]
    terms = 0.5 * theta[fin, 1] ** 2 + abs(math.log(mass)) + abs(math.log(mu_w)) + 1.0
    _within(got[fin], ref[fin], 1e-12 * np.abs(ref[fin]) + 1e-13 * terms, 'logprior')


# ------------------------------------------------------------------------------ g-and-k
@pytest.mark.parametrize('B,n_obs', [(300, 1), (300, 2), (300, 7), (300, 50), (300, 51),
                                     (40000, 128)])
def test_sim_gnk_matches_replay(B, n_obs):
    """Per-row parameters over the prior box; B * ceil(n_obs / 2) = 2.56e6 pairs in the last case,
    above the grid cap of sm_count * 64 blocks of 256 threads, so the grid-stride loop runs."""
    from elfi_b200 import ops
    rs = np.random.RandomState(n_obs)
    A, Bs, g, k = (rs.uniform(0, 10, B) for _ in range(4))
    Bs[0], g[0], k[0] = 10.0, 0.0, 0.0
    seed, offset = 2 ** 32 + 21, 2 ** 32 - 1
    Y = _np(ops.sim_gnk(A, Bs, g, k, n_obs=n_obs, seed=seed, offset=offset))
    Yr, err = streams.sim_gnk(A, Bs, g, k, 0.8, n_obs, seed, offset)
    _within(Y, Yr, err, 'Y')


# ------------------------------------------------------------------------------ mixture CDF
def _weights(kind, N, rs):
    if kind == 'none':
        return None
    if kind == 'zeros':
        w = rs.rand(N) ** 8
        w[rs.rand(N) < 0.3] = 0.0
        w[rs.randint(0, N, 3)] = 0.0
        if N > 40:
            w[10:30] = 0.0                       # a run of zeros
    else:
        w = rs.rand(N) * 10.0 ** rs.randint(-10, 10, N)
    if not w.any():
        w[-1] = 1.0
    return w


CDF_CASES = [(N, kind) for N in (1, 1023, 1024, 1025, 5000, 1000000) for kind in ('zeros', 'mixed', 'none')]


@pytest.mark.parametrize('N,kind', CDF_CASES)
def test_gm_cdf_nondecreasing_and_accurate(N, kind):
    from elfi_b200 import ops
    rs = np.random.RandomState(N)
    w = _weights(kind, N, rs)
    cumw = _np(ops.gm_cdf(w, N))
    ref = np.cumsum(np.ones(N) if w is None else w)
    assert np.all(np.diff(cumw) >= 0), '{} decreasing steps'.format(int(np.sum(np.diff(cumw) < 0)))
    np.testing.assert_allclose(cumw, ref, rtol=1e-12, atol=0)
    total = float(N) if w is None else math.fsum(w)
    assert abs(cumw[-1] - total) <= 1e-13 * total
    if w is not None:
        z = np.flatnonzero(w[1:] == 0) + 1
        assert np.array_equal(cumw[z], cumw[z - 1])      # a zero weight gets no share at all


@pytest.mark.parametrize('N,kind', CDF_CASES)
def test_gm_cdf_equals_replay(N, kind):
    """The table is the kernel's fixed order of additions and maxima, bit for bit."""
    from elfi_b200 import ops
    w = _weights(kind, N, np.random.RandomState(N))
    cumw = _np(ops.gm_cdf(w, N))
    assert np.array_equal(cumw, streams.gm_cdf(w, N))


# ------------------------------------------------------------------------------ mixture proposals
def _spd(rs, p, scale):
    a = rs.randn(p, p)
    return scale * (a @ a.T / p + 0.5 * np.eye(p))


def _run_gm(means_host, cov, w, B, seed, offset, support, box=None, ld_pad=3):
    """gm_rvs on the device (means as a row-strided view with ldm = p + ld_pad) and the replay
    driven by the device's own CDF table."""
    import torch
    from elfi_b200 import ops
    N, p = means_host.shape
    store = torch.zeros((N, p + ld_pad), dtype=torch.float64, device='cuda')
    store[:, :p] = torch.from_numpy(means_host).cuda()
    means = store[:, :p]
    cdf = ops.gm_cdf(w, N)
    x = _np(ops.gm_rvs(means, cov, None, B, seed=seed, offset=offset, support=support, box=box, cdf=cdf))
    L = np.linalg.cholesky(np.atleast_2d(cov))
    xr, trial, comp, err, margin = streams.gm_rvs(means_host, L, _np(cdf), B, seed, offset, support, box)
    return x, xr, trial, comp, err, margin


def _check_gm(x, xr, trial, err, margin, w):
    amb = margin < 1e-9               # a decision near a boundary could go either way in ulps
    assert amb.sum() <= max(2, 1e-4 * x.shape[0]), int(amb.sum())
    _within(x[~amb], xr[~amb], err[~amb, None], 'draws')
    return amb


GM_CASES = [(p, N, support) for p in (1, 2, 3, 4) for N in (1, 500, 1000000) for support in (0, 2)] + \
           [(2, N, 1) for N in (1, 500, 1000000)]


@pytest.mark.parametrize('p,N,support', GM_CASES)
def test_gm_rvs_matches_replay(p, N, support):
    rs = np.random.RandomState(p * 10 + support + N % 7)
    B = 20000
    if support == 1:
        # components near the edges of the MA2 support: many rows need a second trial or more
        t1 = rs.uniform(-1.95, 1.95, N)
        means = np.column_stack([t1, np.where(rs.rand(N) < 0.5, 0.97, -0.97 + np.abs(t1))])
        cov = np.array([[0.01, 0.002], [0.002, 0.004]])
        box = None
    else:
        means = rs.uniform(-1, 1, (N, p))
        means[0] = 0.8                         # on the box's upper faces
        cov = _spd(rs, p, 0.05)
        box = (np.full(p, -1.0), np.full(p, 0.8)) if support == 2 else None
    w = rs.rand(N) ** 4
    if N > 2:
        w[0] = w[-1] = 0.0
        w[rs.randint(1, N - 1, max(1, N // 10))] = 0.0
    x, xr, trial, comp, err, margin = _run_gm(means, cov, w, B, 2 ** 32 + 9, 2 ** 32 - 7, support, box)
    _check_gm(x, xr, trial, err, margin, w)
    assert np.all(w[comp] > 0)                 # zero-weight components are never drawn
    assert np.all(trial >= 0)
    if support != 0:
        assert np.sum(trial >= 1) > 0.05 * B   # the redraw path is exercised
        assert np.sum(trial >= 3) > 0
    if support == 2:
        assert np.all((x >= box[0]) & (x <= box[1]))


def test_gm_rvs_all_trials_rejected_returns_last_draw():
    """A box apart from the mixture: after 1000 rejected draws the kernel returns the 1000th
    (documented in include/elfi_b200.h); pinned against the replay."""
    rs = np.random.RandomState(3)
    means = rs.uniform(-0.1, 0.1, (5, 3))
    cov = np.eye(3) * 0.01
    box = (np.full(3, 10.0), np.full(3, 11.0))
    x, xr, trial, comp, err, margin = _run_gm(means, cov, np.ones(5), 64, 17, 0, 2, box)
    assert np.all(trial == -1)
    _within(x, xr, err[:, None], 'draws of trial 999')
    assert np.all(x < 10.0)
