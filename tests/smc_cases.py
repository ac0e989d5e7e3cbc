"""Accuracy checks of the SMC population arithmetic of smc.cu against plain high-precision
references; the case bodies shared by test_smc_accuracy_gpu.py (the device) and
test_smc_accuracy_cpu_double.py (the CPU test double, which rehearses the references, the bounds
and the shape plumbing without a GPU).

Mixture density (elfi_b200_gm_logpdf_f64 / _mixed_f64, through ops.gm_logpdf)
--------------------------------------------------------------------------
Reference.  `mixture_reference` evaluates log q(x) = lognorm + log sum_j w_j exp(-maha_j / 2) in
fp64 from DIRECT differences d = x - m_j (not the kernel's expanded, centred form), whitened with
the same Linv and log-determinant that ops.gm_logpdf hands to the kernel (so the conditioning of
the covariance does not enter the comparison), and with the largest term factored out
(log-sum-exp).  maha = |Linv d|^2 carries a relative error of about (p + 3) 2^-53, an absolute
error of (maha / 2) (p + 3) 2^-53 in the log of a term; the shifted sum adds log2(M) 2^-53
relative.  Its error is therefore about (maha / 2 + log2 M) 2^-53 relative -- 1e-13 at maha ~
1400 and p = 2, 1.5e-12 at p = 16 -- three orders or more below every bound tested here
(test_gm_formula_host.py checks it against mpmath at 40 digits).  Per point it also reports
  * `dev_flush`: every term lies below 2^-1020 (nt > 1020), where the kernel flushes to zero,
  * `scipy_underflow`: every term underflows in the reference's exp(lognorm - maha / 2), and
  * `lost`: the share of q held by terms that either convention may drop or evaluate in the
    subnormal range (nt > 1020 - 1e-6, or lognorm - maha / 2 < -708).

Bounds.  Every term is positive, so the relative error of q is at most the largest relative term
error plus the fp64 accumulation (chunk length + chunk count) 2^-53 < 2e-12.
  fp64 path: the degree-6 minimax 2^f is within 1.9e-9 of 2^f on [-.5, .5] (test_gm_formula_host.py
    checks the shipped exp2_neg against mpmath); f = -nt - rint(-nt) and the exponent insertion
    are exact; nt carries the cancellation error of the expanded distance, (p + 2) 2^-53 |y|^2
    absolute: < 1e-13 for SMC clouds centred at one of their points, 2e-10 (ln 2 times that,
    relative) with means[0] an outlier at 1e3 proposal standard deviations.  log, lognorm and the
    reference add < 2e-12.  So 1.9e-9 + 2e-10 + 4e-12 < FP64_BOUND = 5e-9, half the 1e-8 that
    include/elfi_b200.h promises, and the bound test_gm_formula_host.py assumes for the same
    arithmetic on the host.
  mixed path: 2^f from ex2.approx.ftz.f32, which the PTX ISA states to be within 2 ulp of 2^f
    over the full range: 2^-22 = 2.38e-7 relative for a result just above 1.0, where an fp32 ulp
    is 2^-23; f itself is rounded to fp32 (|f| <= .5: <= 2^-26 absolute, ln 2 2^-26 = 1.0e-8
    relative in 2^f); the widening to fp64 is exact.  MIXED_BOUND = 2^-22 + ln 2 2^-26 + 1e-9
    (the fp64 part above) = 2.50e-7.
Underflow contract.  Where `lost` is below 1 % of the bound: finite and within the bound.  Where
every term both flushes and underflows: -inf.  Points in between -- the kernel flushes below
2^-1020 and adds the normaliser after the log, the reference underflows below 2^-1074 with the
normaliser inside the exp -- are counted and reported, not asserted.

Invariance (bit for bit): slicing the point batch (including the shards sharding.shard_bounds
cuts, which the multi-GPU density relies on: the component chunk length depends on M only),
permuting the points, repeating a call, weights=np.ones(M) against weights=None, row-strided
inputs against contiguous ones, and mixed=True against the fp64 path on the generic kernel
(p >= 5, which has no mixed variant).

Kernel paths by shape: p <= 4 runs gm_pdf_kernel<p> with component chunks of
clamp(512 ceil((M / 64) / 512), 2048, 16384) components, 512-component shared-memory tiles and
512-point blocks; 5 <= p <= 16 runs gm_pdf_generic_kernel, one point per thread over all M.
  M = 1, 511, 512, 513       one chunk; no full tile, one tile, a one-component tile tail
  M = 2048, 2049             one chunk exactly; two chunks, the last of one component
  M = 3000                   two chunks (2048 + 952)
  M = 131073                 chunk 2048, 65 chunks, the last of one component
  M = 1_000_000              chunk 15872, 64 chunks, the last of 64 components (the production shape)
  M = 2_097_153              the 16384 clamp: 129 chunks, the last of one component
  N = 0, 1, 3, 5, 511, 513, 1777   point-block tails (512 points per block)

Weighted statistics (elfi_b200_weighted_stats_f64)
--------------------------------------------------
Reference: two passes in np.longdouble (V1, V2, xbar, then sum w (x - xbar)^2 about the
reference's own xbar); with fewer than two nonzero weights V1 - V2 / V1 is exactly zero, so the
reference s2 is 0 / 0.  Bound: the device sums each quantity through a tree of depth
  d = ceil(N / (blocks 256)) (per-thread stride) + 5 (warp) + 8 (block) + blocks (final),
  blocks = min(ceil(N / 256), 4 SMs),
so |error| <= d u sum |terms|, u = 2^-53 (each term enters through d roundings; an fma adds one).
  V1, V2: d u V1, d u V2 (terms >= 0).
  xbar_j = S_j / V1: d u (A_j + |S_j|) / V1 + u |xbar_j|, A_j = sum |w x_j|; relative to
    |xbar_j| that is d u (kappa + 1) + u with the condition number kappa = A_j / |S_j|.
  num_j = sum w (x - xbar_dev)^2: each term 3u (difference, square, fma), the sum d u, and the
    device's xbar error dx adds exactly dx^2 V1 (the cross term sum w (x - xbar) vanishes).
  D = V1 - V2 / V1: d u V1 + (2 d + 1) u V2 / V1 + u |D|.
  s2 = num / D: the relative errors add, plus u.
Every check allows C = 2 times its first-order bound.  Where the bound reaches the value itself (no
significant digit left, e.g. one weight 1e16 times all others) only non-finiteness is compared.

smc_weights: within 2 ulp of np.exp(logprior - logq) (CUDA's exp is within 1 ulp, NumPy's within
1), with NumPy's 0, inf and NaN for -inf arguments.
"""
import math
import types

import numpy as np
import pytest
import torch

from elfi_b200 import _lib, ops, sharding
from elfi_b200 import device as dev

U = 2.0 ** -53
LN2 = math.log(2.0)
FP64_BOUND = 5e-9
HEADER_FP64_BOUND = 1e-8
MIXED_BOUND = 2.0 ** -22 + LN2 * 2.0 ** -26 + 1e-9
WS_C = 2.0
REF_PAIRS = 1.5e8          # host reference budget per case (pairs of point and component)
MEASURED = {}              # largest relative error seen per mode (reported by the GPU module)


def _note(key, value):
    MEASURED[key] = max(MEASURED.get(key, 0.0), float(value))


# ---------------------------------------------------------------------------- mixture reference
def full_cov(cov, p):
    """The covariance matrix ops.gm_logpdf builds from `cov` (a scalar means cov * I)."""
    cov = np.atleast_2d(np.asarray(cov, dtype=np.float64))
    return np.eye(p) * cov[0, 0] if cov.shape == (1, 1) and p > 1 else cov


def mixture_reference(x, means, cov, w=None):
    """Per point: exact log q, the share of q that a convention may lose (`lost`), and whether
    every term flushes on the device (`dev_flush`) or underflows SciPy-style (`scipy_underflow`)."""
    M, p = means.shape
    L = np.linalg.cholesky(full_cov(cov, p))
    Linv = np.linalg.inv(L)
    lognorm = -0.5 * (p * 1.8378770664093453 + 2.0 * float(np.sum(np.log(np.diag(L)))))
    wn = np.full(M, 1.0 / M) if w is None else np.asarray(w, dtype=np.float64) / np.sum(w)
    with np.errstate(divide='ignore'):
        logw = np.log(wn)
    n = len(x)
    logq, lost = np.empty(n), np.empty(n)
    dev_flush, scipy_underflow = np.empty(n, dtype=bool), np.empty(n, dtype=bool)
    b = max(1, int(4e6 // M))
    flush_a = -(1020.0 - 1e-6) * LN2       # a = log(w exp(-maha / 2)) = -nt ln 2
    surely_flushed = -(1020.0 + 1e-6) * LN2
    for lo in range(0, n, b):
        d = x[lo:lo + b, None, :] - means[None, :, :]
        z = d @ Linv.T
        maha = np.einsum('ijk,ijk->ij', z, z)
        a = logw[None, :] - 0.5 * maha
        amax = a.max(axis=1, keepdims=True)
        with np.errstate(under='ignore'):
            e = np.exp(a - amax)
        s = e.sum(axis=1)
        logq[lo:lo + b] = lognorm + amax[:, 0] + np.log(s)
        scipy_e = lognorm - 0.5 * maha
        risky = (a < flush_a) | (scipy_e < -708.0)
        lost[lo:lo + b] = np.where(risky, e, 0.0).sum(axis=1) / s
        dev_flush[lo:lo + b] = np.all(a < surely_flushed, axis=1)
        scipy_underflow[lo:lo + b] = np.all((scipy_e < -746.0) | (wn[None, :] == 0), axis=1)
    return types.SimpleNamespace(logq=logq, lost=lost, dev_flush=dev_flush,
                                 scipy_underflow=scipy_underflow, lognorm=lognorm)


def sample_rows(N, M, k=None, seed=0):
    """Rows the host reference covers: all of them when N * M fits REF_PAIRS (or N <= k), else
    the first 64, the last 64 (at N = 1e6 exactly the last, partial 512-point block) and random
    rows between, k in all."""
    k = max(int(REF_PAIRS // M), 128) if k is None else k
    if N <= k:
        return np.arange(N)
    rs = np.random.RandomState(seed)
    mid = rs.choice(np.arange(64, N - 64), size=k - 128, replace=False)
    return np.unique(np.concatenate([np.arange(64), mid, np.arange(N - 64, N)]))


def gm(x, means, cov, w=None, mixed=False):
    return ops.gm_logpdf(x, means, cov, w, mixed=mixed).cpu().numpy()


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


def check_against(got, ref, mixed, tag, min_checked=0.5):
    """got (device, at the reference's rows) against the reference under the underflow contract.
    Returns (max relative error, checked, both-underflow, in-between counts)."""
    bound = MIXED_BOUND if mixed else FP64_BOUND
    ok = ref.lost <= 0.01 * bound
    both = ref.dev_flush & ref.scipy_underflow
    between = ~ok & ~both
    assert np.all(np.isfinite(got[ok])), '{}: non-finite where q is representable'.format(tag)
    with np.errstate(invalid='ignore'):
        err = np.abs(np.expm1(got[ok] - ref.logq[ok]))
    worst = float(err.max()) if err.size else 0.0
    _note('mixed' if mixed else 'fp64', worst)
    bad = np.nonzero(~(err <= bound))[0]
    assert bad.size == 0, '{}: {} of {} points beyond {:.3g}, worst {:.3g} at row {}'.format(
        tag, bad.size, err.size, bound, worst, np.nonzero(ok)[0][bad[0]])
    if not mixed:
        assert worst <= HEADER_FP64_BOUND
    assert np.all(got[both] == -np.inf), '{}: finite where every term underflows'.format(tag)
    assert ok.sum() >= min_checked * len(got), '{}: only {} of {} points checkable'.format(
        tag, ok.sum(), len(got))
    print('{}: max rel err {:.3g} (bound {:.3g}) over {} points; {} -inf; {} in the band'.format(
        tag, worst, bound, int(ok.sum()), int(both.sum()), int(between.sum())))
    return worst, int(ok.sum()), int(both.sum()), int(between.sum())


# ---------------------------------------------------------------------------- data
COV_KINDS = ['scalar', 'diag', 'full', 'cond1e8', 'var1e-8', 'var1e4']
W_KINDS = ['none', 'ones', 'cube', 'smc', 'tenth_zero', 'one']


def make_cov(kind, p, rs):
    if kind == 'scalar':
        return 0.3                                   # cov * I
    if kind == 'diag':
        return np.diag(2.0 * rs.uniform(0.05, 2.0, p) ** 2)     # 2 diag(weighted var), as SMC
    if kind == 'full':
        A = rs.randn(p, p)
        return A @ A.T / p + 0.1 * np.eye(p)
    if kind == 'cond1e8':
        Q, _ = np.linalg.qr(rs.randn(p, p))
        return (Q * np.logspace(-4, 4, p)) @ Q.T if p > 1 else np.array([[1e-4]])
    if kind == 'var1e-8':
        return np.diag(1e-8 * rs.uniform(0.5, 2.0, p))          # lognorm > 0
    if kind == 'var1e4':
        return np.diag(1e4 * rs.uniform(0.5, 2.0, p))           # lognorm < 0
    raise ValueError(kind)


def single_weight_value(rs):
    """A weight w whose rounded w^2 / w is not w (one in ~13 doubles): with it as the only nonzero
    weight the naive V1 - V2 / V1 is an ulp instead of zero."""
    while True:
        v = rs.uniform(0.5, 2.0)
        if (v * v) / v != v:
            return v


def make_weights(kind, M, rs):
    if kind == 'none':
        return None
    if kind == 'ones':
        return np.ones(M)
    if kind == 'cube':
        return rs.rand(M) ** 3
    if kind == 'smc':
        return np.exp(15.0 * rs.randn(M))            # ~1e-30 .. 1e30
    if kind == 'tenth_zero':
        w = rs.rand(M)
        w[9::10] = 0.0
        return w
    if kind == 'one':
        w = np.zeros(M)
        w[M // 2] = single_weight_value(rs)
        return w
    raise ValueError(kind)


def cloud(M, N, p, cov, rs, loc=0.0, far=0):
    """SMC-like population: means spread like the proposal / 2, points = a mean plus a proposal
    draw, and `far` points 5 .. 50 proposal standard deviations out (the underflow band)."""
    G = np.linalg.cholesky(full_cov(cov, p))
    means = loc + rs.randn(M, p) @ G.T / np.sqrt(2.0)
    x = means[rs.randint(0, M, N)] + rs.randn(N, p) @ G.T
    if far:
        u = rs.randn(far, p)
        u /= np.linalg.norm(u, axis=1, keepdims=True)
        x[:far] = loc + (u * np.linspace(5.0, 50.0, far)[:, None]) @ G.T
    return means, x


def modes(p):
    return (False, True) if p <= 4 else (False,)


def check_case(x, means, cov, w, tag, rows=None, min_checked=0.5):
    """Both modes (p <= 4) against one reference; for p >= 5 mixed must equal fp64 bit for bit."""
    N, M, p = len(x), len(means), means.shape[1]
    rows = sample_rows(N, M) if rows is None else rows
    ref = mixture_reference(x[rows], means, cov, w)
    out = {}
    for mixed in modes(p):
        got = gm(x, means, cov, w, mixed)
        assert got.shape == (N,)
        check_against(got[rows], ref, mixed, '{} {}'.format(tag, 'mixed' if mixed else 'fp64'),
                      min_checked)
        out[mixed] = got
    if p > 4:
        assert same_bits(gm(x, means, cov, w, True), out[False]), tag + ': generic mixed != fp64'
    return out, ref, rows


# ---------------------------------------------------------------------------- mixture cases
TEMPLATED_P = [1, 2, 3, 4]
GENERIC_P = [5, 8, 16]
CHUNK_M = [1, 511, 512, 513, 2048, 2049, 3000, 131073, 2_097_153]   # + 1_000_000: case_production
TAIL_N = [0, 1, 3, 5, 511, 513, 1777]
CENTRING_SD = [1e1, 1e2, 1e3]


def case_templated(p):
    rs = np.random.RandomState(100 + p)
    cov = make_cov('full', p, rs)
    means, x = cloud(3000, 1777, p, cov, rs, loc=rs.uniform(-3, 3, p), far=40)
    check_case(x, means, cov, make_weights('cube', 3000, rs), 'templated p={}'.format(p))


def case_generic(p):
    rs = np.random.RandomState(200 + p)
    cov = make_cov('full', p, rs)
    means, x = cloud(4096, 4096, p, cov, rs, far=40)
    check_case(x, means, cov, make_weights('cube', 4096, rs), 'generic p={}'.format(p))


def case_p17_rejected():
    """p = 17 is refused (no kernel has room for it), and the context still works afterwards."""
    rs = np.random.RandomState(17)
    means, x = rs.randn(50, 17), rs.randn(20, 17)
    with pytest.raises(_lib.ElfiB200Error, match='p <= 16'):
        gm(x, means, np.eye(17))
    cov = make_cov('full', 3, rs)
    m3, x3 = cloud(600, 300, 3, cov, rs)
    check_case(x3, m3, cov, None, 'after p=17')


def case_chunking(M, p=2):
    rs = np.random.RandomState(M % 100003)
    cov = make_cov('diag', p, rs)
    means, x = cloud(M, 1777, p, cov, rs, far=20)
    check_case(x, means, cov, make_weights('cube', M, rs), 'chunks M={} p={}'.format(M, p))


def case_point_tails(N, p=3):
    rs = np.random.RandomState(300 + N)
    cov = make_cov('full', p, rs)
    means, x = cloud(3000, max(N, 1), p, cov, rs)
    x = x[:N]
    if N == 0:
        for mixed in (False, True):
            assert gm(x, means, cov, None, mixed).shape == (0,)
        return
    check_case(x, means, cov, None, 'tails N={}'.format(N), min_checked=1.0)


def case_covariance(kind, p):
    rs = np.random.RandomState(400 + 10 * p + COV_KINDS.index(kind))
    cov = make_cov(kind, p, rs)
    means, x = cloud(3000, 1777, p, cov, rs, loc=rs.uniform(-5, 5, p), far=40)
    check_case(x, means, cov, make_weights('cube', 3000, rs), 'cov {} p={}'.format(kind, p))


def case_weights(kind, p=2):
    rs = np.random.RandomState(500 + W_KINDS.index(kind))
    cov = make_cov('diag', p, rs)
    M = 3000
    means, x = cloud(M, 1777, p, cov, rs, far=40)
    w = make_weights(kind, M, rs)
    # a single component leaves most points far out in its tails
    out, _, _ = check_case(x, means, cov, w, 'weights {}'.format(kind),
                           min_checked=0.2 if kind == 'one' else 0.5)
    if kind == 'ones':
        for mixed in (False, True):
            assert same_bits(out[mixed], gm(x, means, cov, None, mixed)), 'ones != None'


def case_centring(sd, p=2):
    """means[0] an outlier `sd` proposal standard deviations away from the rest of the cloud."""
    rs = np.random.RandomState(600 + int(np.log10(sd)))
    cov = make_cov('diag', p, rs)
    means, x = cloud(3000, 1777, p, cov, rs, loc=1.0)
    G = np.linalg.cholesky(cov)
    means[0] = 1.0 + sd * (np.ones(p) / np.sqrt(p)) @ G.T
    check_case(x, means, cov, make_weights('cube', 3000, rs), 'centring {:g} sd'.format(sd))


def _strided(A, ld, offset, rs):
    """Device view of A with leading dimension ld, starting `offset` rows into its buffer."""
    buf = rs.randn(len(A) + offset, ld) * 1e3          # garbage around the view
    buf[offset:, :A.shape[1]] = A
    return dev.to_device(buf)[offset:, :A.shape[1]]


def case_strided(p):
    rs = np.random.RandomState(700 + p)
    cov = make_cov('full', p, rs)
    means, x = cloud(2049, 777, p, cov, rs)
    w = make_weights('cube', 2049, rs)
    xv = _strided(x, p + 3, 1, rs)
    mv = _strided(means, p + 5, 3, rs)
    assert xv.stride(0) == p + 3 and mv.stride(0) == p + 5
    out, _, _ = check_case(x, means, cov, w, 'strided contiguous p={}'.format(p))
    for mixed in modes(p):
        assert same_bits(gm(xv, mv, cov, w, mixed), out[mixed]), 'strided != contiguous'


def case_underflow(p, cov_kind):
    """Points from inside the cloud out to 50 standard deviations: the bulk within the bound,
    the far points -inf, the band between counted."""
    rs = np.random.RandomState(800 + p)
    cov = make_cov(cov_kind, p, rs)
    means, x = cloud(3000, 1500, p, cov, rs, far=1200)
    rows = np.arange(len(x))
    ref = mixture_reference(x, means, cov, None)
    both = ref.dev_flush & ref.scipy_underflow
    assert both.sum() > 0 and (ref.lost <= 0.01 * FP64_BOUND).sum() > 300
    for mixed in modes(p):
        got = gm(x, means, cov, None, mixed)
        check_against(got[rows], ref, mixed, 'underflow p={} {} {}'.format(
            p, cov_kind, 'mixed' if mixed else 'fp64'), min_checked=0.2)


SLICES = [(0, 1), (1, 2), (3, 515), (511, 1025), (777, 1777), (1, 1777), (1000, 1001)]


def case_invariance(p):
    """Slices, permutations and repeated calls give the same bits; permuting the components
    (means[0] excepted: it is the centre) stays within the bound."""
    rs = np.random.RandomState(900 + p)
    cov = make_cov('full', p, rs)
    M, N = 3000, 1777
    means, x = cloud(M, N, p, cov, rs, far=20)
    w = make_weights('smc', M, rs)
    xd = dev.to_device(x)
    ref = mixture_reference(x, means, cov, w)
    for mixed in modes(p):
        tag = 'invariance p={} {}'.format(p, 'mixed' if mixed else 'fp64')
        full = gm(xd, means, cov, w, mixed)
        assert same_bits(gm(xd, means, cov, w, mixed), full), tag + ': repeat'
        for lo, hi in SLICES:
            assert same_bits(gm(xd[lo:hi], means, cov, w, mixed), full[lo:hi]), \
                '{}: slice {}:{}'.format(tag, lo, hi)
        perm = rs.permutation(N)
        assert same_bits(gm(x[perm], means, cov, w, mixed), full[perm]), tag + ': point perm'
        cperm = np.concatenate([[0], 1 + rs.permutation(M - 1)])
        got = gm(x, means[cperm], cov, w[cperm], mixed)
        check_against(got, ref, mixed, tag + ' component perm')


def case_production(p=2):
    """M = N = 1e6 (64 chunks of 15872, a last chunk of 64 components): reference on 256 rows
    against all components, and the shards of the batch bit for bit."""
    rs = np.random.RandomState(1000 + p)
    M = N = 1_000_000
    cov = make_cov('diag', p, rs)
    means, x = cloud(M, N, p, cov, rs, loc=0.5, far=64)
    w = make_weights('cube', M, rs)
    rows = sample_rows(N, M, k=256)
    assert len(rows) == 256 and rows[-1] == N - 1
    out, _, _ = check_case(x, means, cov, w, 'production', rows=rows)
    xd, md, wd = dev.to_device(x), dev.to_device(means), dev.to_device(w)
    for mixed, worlds in ((False, (3, 8)), (True, (8,))):
        for size in worlds:
            for rank in range(size):
                lo, hi, _ = sharding.shard_bounds(N, rank, size)
                got = ops.gm_logpdf(xd[lo:hi], md, cov, wd, mixed=mixed).cpu().numpy()
                assert same_bits(got, out[mixed][lo:hi]), 'shard {}/{} mixed={}'.format(
                    rank, size, mixed)


# ---------------------------------------------------------------------------- weighted stats
def sm_count():
    if torch.cuda.is_available():
        return torch.cuda.get_device_properties(0).multi_processor_count
    return 132                                        # H100 SXM; the CPU double has no SMs


def ws_depth(N):
    blocks = min((N + 255) // 256, 4 * sm_count())
    return -(-N // (blocks * 256)) + 5 + 8 + blocks


def ws_reference(x, w):
    ld = np.longdouble
    X = x.astype(ld)
    W = np.ones(len(x), dtype=ld) if w is None else w.astype(ld)
    V1, V2 = W.sum(), (W * W).sum()
    S = W @ X
    A = np.abs(W) @ np.abs(X)
    with np.errstate(all='ignore'):
        xbar = S / V1
        num = W @ ((X - xbar) ** 2)
        nz = len(x) if w is None else np.count_nonzero(w)
        D = V1 - V2 / V1 if nz > 1 else ld(0)
        s2 = num / D
    return types.SimpleNamespace(V1=V1, V2=V2, S=S, A=A, xbar=xbar, num=num, D=D, s2=s2)


def ws_check(x, w, tag, xv=None):
    N, p = x.shape
    V1, V2, xbar, s2 = ops.weighted_stats(x if xv is None else xv, w)
    r = ws_reference(x, w)
    d = ws_depth(N)
    f = lambda v: np.asarray(v, dtype=np.float64)                       # noqa: E731
    with np.errstate(all='ignore'):
        V1r, V2r, Dr = np.float64(r.V1), np.float64(r.V2), np.float64(r.D)
        b_xbar = d * U * (f(r.A) + np.abs(f(r.S))) / V1r + U * np.abs(f(r.xbar))
        b_D = d * U * V1r + (2 * d + 1) * U * V2r / V1r + U * abs(Dr)
        rel_num = (d + 3) * U + (WS_C * b_xbar) ** 2 * V1r / np.abs(f(r.num))
        b_s2 = (rel_num + b_D / abs(Dr) + U) * np.abs(f(r.s2))
    checks = [('V1', V1, f(r.V1), d * U * V1r), ('V2', V2, f(r.V2), d * U * V2r),
              ('xbar', xbar, f(r.xbar), b_xbar), ('s2', s2, f(r.s2), b_s2)]
    for name, got, ref, bound in checks:
        got, ref, bound = (np.atleast_1d(np.asarray(v, dtype=np.float64)) for v in (got, ref, bound))
        fin = np.isfinite(ref)
        assert np.all(~np.isfinite(got[~fin])), '{} {}: finite where the reference is not'.format(
            tag, name)
        sig = fin & (WS_C * bound < np.abs(ref))       # the value has significant digits left
        err = np.abs(got[sig] - ref[sig])
        assert np.all(err <= WS_C * bound[sig]), '{} {}: err {} bound {}'.format(
            tag, name, err, WS_C * bound[sig])


WS_P = [1, 2, 3, 4, 7, 16]
WS_N = [1, 2, 255, 256, 257, 4097, 4 * 132 * 256 + 1, 1_000_003]


def case_weighted_stats(p, N, kind='cube'):
    rs = np.random.RandomState(p * 1000 + N % 997 + W_KINDS.index(kind))
    x = rs.randn(N, p) * rs.uniform(0.1, 10.0, p) + rs.uniform(-5, 5, p)
    ws_check(x, make_weights(kind, N, rs), 'wstats p={} N={} {}'.format(p, N, kind))


def case_weighted_stats_offset(N=1_000_003, p=2):
    """x offset by 1e6 with spread 1: xbar well conditioned, s2 from small differences."""
    rs = np.random.RandomState(31)
    x = 1e6 + rs.randn(N, p)
    ws_check(x, make_weights('smc', N, rs) if N > 1 else None, 'wstats offset N={}'.format(N))
    ws_check(x, None, 'wstats offset unweighted N={}'.format(N))


def case_weighted_stats_strided(p=4, N=4097):
    rs = np.random.RandomState(37)
    x = rs.randn(N, p) + 3.0
    w = make_weights('cube', N, rs)
    xv = _strided(x, p + 3, 1, rs)
    ws_check(x, w, 'wstats strided', xv=xv)
    a = ops.weighted_stats(xv, w)
    b = ops.weighted_stats(x, w)
    assert all(same_bits(np.atleast_1d(u), np.atleast_1d(v)) for u, v in zip(a, b))


# ---------------------------------------------------------------------------- smc_weights
def case_smc_weights():
    rs = np.random.RandomState(41)
    n = 100_003
    lp = rs.uniform(-350, 350, n)
    lq = rs.uniform(-350, 350, n)
    lp[:3] = [-np.inf, 1.0, -np.inf]
    lq[:3] = [2.0, -np.inf, -np.inf]
    got = ops.smc_weights(lp, lq).cpu().numpy()
    ref = np.exp(lp - lq)
    assert got[0] == 0.0 and got[1] == np.inf and np.isnan(got[2])
    fin = np.isfinite(ref)
    assert np.array_equal(np.isnan(got), np.isnan(ref)) and np.array_equal(got[~fin & ~np.isnan(ref)],
                                                                           ref[~fin & ~np.isnan(ref)])
    assert np.all(np.abs(got[fin] - ref[fin]) <= 2 * np.spacing(ref[fin]))
