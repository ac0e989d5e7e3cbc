"""CPU check of the arithmetic of the mixture-density kernel (elfi_b200/csrc/smc.cu, gm_pdf_kernel):
the per-term 2^(-nt) is the shipped exp2_neg of elfi_b200/csrc/gmterm.cuh, built for the host by
tests/harness/gmterm_harness.cpp and checked against mpmath (< 1.9e-9 relative per term, exact
flush above nt = 1020); the centred / expanded squared distance with the folded log-weight is
restated in NumPy around it and compared with a float128 evaluation of GMDistribution.logpdf
(elfi/methods/utils.py:174-197).  The fp64 mixture reference of tests/smc_cases.py, which the
device accuracy tests compare against, is itself checked against mpmath here."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SCALE = 0.8493218002880191   # sqrt(log2(e) / 2)
TERM_BOUND = 1.9e-9          # relative error per term, include/elfi_b200.h


@pytest.fixture(scope='module')
def harness(tmp_path_factory):
    gxx = shutil.which('g++')
    if gxx is None:
        pytest.skip('g++ not available')
    so = str(tmp_path_factory.mktemp('gmterm') / 'gmterm_harness.so')
    subprocess.check_call([gxx, '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-o',
                           so, os.path.join(HERE, 'harness', 'gmterm_harness.cpp')])
    return ctypes.CDLL(so)


def exp2_neg(lib, nt):
    nt = np.ascontiguousarray(nt, dtype=np.float64)
    out = np.empty_like(nt)
    lib.harness_exp2_neg(nt.ctypes.data_as(ctypes.c_void_p), ctypes.c_int64(nt.size),
                         out.ctypes.data_as(ctypes.c_void_p))
    return out


def kernel_logpdf(lib, x, means, cov, w):
    L = np.linalg.cholesky(cov)
    Linv = np.linalg.inv(L)
    p = x.shape[1]
    centre = means[0]
    y = (x - centre) @ Linv.T * SCALE
    m = (means - centre) @ Linv.T * SCALE
    with np.errstate(divide='ignore'):
        cj = np.sum(m * m, axis=1) - np.log2(w / w.sum())
    g = cj[None, :] + y @ (-2.0 * m).T
    nt = g + np.sum(y * y, axis=1)[:, None]
    acc = exp2_neg(lib, nt).sum(axis=1)
    lognorm = -0.5 * (p * np.log(2 * np.pi) + 2 * np.sum(np.log(np.diag(L))))
    return np.log(acc) + lognorm


def exact_logpdf(x, means, cov, w):
    ld = np.longdouble
    prec = np.linalg.inv(cov).astype(ld)
    d = x[:, None, :].astype(ld) - means[None, :, :].astype(ld)
    maha = np.einsum('ijk,kl,ijl->ij', d, prec, d)
    wn = (w / w.sum()).astype(ld)
    p = x.shape[1]
    dens = (wn[None, :] * np.exp(-maha / 2)).sum(axis=1)
    return (np.log(dens) - ld(0.5) * (p * np.log(ld(2) * np.pi) + np.log(ld(np.linalg.det(cov))))
            ).astype(np.float64)


@pytest.mark.parametrize('p,loc,sd', [(2, 0.5, 0.2), (2, 0.6, 0.004), (1, -3.0, 1.5), (4, 5.0, 0.05),
                                      (3, 1e3, 1e-2), (2, 0.0, 30.0)])
def test_kernel_arithmetic_matches_float128(harness, p, loc, sd):
    rs = np.random.RandomState(p * 7 + int(sd * 1000) % 97)
    M, N = 3000, 400
    means = loc + sd * rs.randn(M, p) * rs.uniform(0.5, 2.0, p)
    w = rs.rand(M) ** 3
    w[::17] = 0.0                                    # zero weights never contribute
    A = rs.randn(p, p) * 0.3 + np.eye(p)
    cov = 2 * sd ** 2 * (A @ A.T)
    x = np.vstack([means[rs.choice(M, N - 40)] + np.sqrt(2) * sd * rs.randn(N - 40, p),
                   loc + 8 * sd * rs.randn(40, p)])  # incl. points far in the tails
    got = kernel_logpdf(harness, x, means, cov, w)
    want = exact_logpdf(x, means, cov, w)
    ok = np.isfinite(want) & (want > -600)
    assert ok.sum() > N // 2
    np.testing.assert_allclose(np.exp(got[ok] - want[ok]), 1.0, rtol=5e-9)


def _mp_exp2_neg(nt):
    import mpmath as mp
    return np.array([float(mp.power(2, -mp.mpf(float(v)))) for v in nt])


def _term_inputs():
    rs = np.random.RandomState(5)
    k = np.arange(0.0, 1020.5, 0.5)              # integers and half-integers: range-reduction edges
    edges = np.concatenate([np.nextafter(k, -np.inf), k, np.nextafter(k, np.inf)])
    edges = edges[edges <= 1020.0]
    return np.concatenate([rs.uniform(0.0, 1020.0, 4000), rs.uniform(0.0, 2.0, 1000), edges,
                           [np.nextafter(1020.0, -np.inf), 1020.0, -1e-14, 0.0, -0.0]])


def test_exp2_neg_against_mpmath(harness):
    """The shipped 2^(-nt): < 1.9e-9 relative everywhere in [0, 1020], including both sides of
    every integer and half-integer (where k and the sign of f switch), 1020 itself and the small
    negative nt that cancellation in the expanded distance can produce."""
    pytest.importorskip('mpmath').mp.dps = 30
    nt = _term_inputs()
    got = exp2_neg(harness, nt)
    want = _mp_exp2_neg(nt)
    rel = np.abs(got / want - 1.0)
    assert rel.max() < TERM_BOUND, (rel.max(), nt[np.argmax(rel)])
    assert rel.max() > 1e-10        # the polynomial's own error is visible: not an exact exp2


def test_exp2_neg_flush_and_non_finite(harness):
    """nt > 1020 flushes to exactly 0 from the first double above 1020 on; +inf (a zero weight)
    and NaN give 0."""
    above = np.array([np.nextafter(1020.0, np.inf), 1020.5, 1021.0, 1074.0, 1100.0, 1e300, np.inf,
                      np.nan])
    got = exp2_neg(harness, above)
    assert np.array_equal(got, np.zeros_like(above))
    assert not np.signbit(got).any()


def test_exp2_neg_dense_sweep(harness):
    """1e6 points over [0, 1020] against NumPy's exp2 (within 1 ulp, 1e7 times below the bound)."""
    nt = np.random.RandomState(6).uniform(-1e-12, 1020.0, 1_000_000)
    got = exp2_neg(harness, nt)
    assert np.abs(got / np.exp2(-nt) - 1.0).max() < TERM_BOUND


def test_mixture_reference_against_mpmath():
    """smc_cases.mixture_reference (fp64, direct differences, log-sum-exp) against a 40-digit
    mpmath evaluation with the same Linv and log-determinant, from the bulk out to maha ~ 1400:
    within 8 (maha / 2 + log2 M + p) 2^-53 relative, the error its docstring derives."""
    mp = pytest.importorskip('mpmath')
    mp.mp.dps = 40
    import smc_cases
    rs = np.random.RandomState(7)
    for p, M in ((1, 5), (2, 7), (4, 3)):
        A = rs.randn(p, p)
        cov = A @ A.T / p + 0.2 * np.eye(p)
        means = rs.randn(M, p)
        w = rs.rand(M)
        L = np.linalg.cholesky(cov)
        Linv = np.linalg.inv(L)
        u = rs.randn(12, p)
        u /= np.linalg.norm(u, axis=1, keepdims=True)
        r = np.concatenate([rs.uniform(0.0, 3.0, 6), np.sqrt([200.0, 600.0, 1000.0, 1300.0,
                                                              1400.0, 1450.0])])
        x = (u * r[:, None]) @ L.T                          # whitened distance r from the origin
        ref = smc_cases.mixture_reference(x, means, cov, w)
        logdet = 2 * sum(mp.log(mp.mpf(v)) for v in np.diag(L))
        lognorm = -(p * mp.log(2 * mp.pi) + logdet) / 2
        W = [mp.mpf(v) for v in w]
        Ws = sum(W)
        for i in range(len(x)):
            terms, mahas = [], []
            for j in range(M):
                d = [mp.mpf(x[i, k]) - mp.mpf(means[j, k]) for k in range(p)]
                z = [sum(mp.mpf(Linv[a, b]) * d[b] for b in range(p)) for a in range(p)]
                maha = sum(v * v for v in z)
                mahas.append(float(maha))
                terms.append(W[j] / Ws * mp.exp(-maha / 2))
            want = lognorm + mp.log(sum(terms))
            err = abs(float(mp.expm1(mp.mpf(ref.logq[i]) - want)))
            tol = 8 * (max(mahas) / 2 + np.log2(M) + p) * 2.0 ** -53
            assert err <= tol, (p, i, err, tol, min(mahas))
        assert max(mahas) > 1000
