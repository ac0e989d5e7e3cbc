"""CPU checks of the throughput-mode generator and of its NumPy replay (oracle/streams.py).

The replay is what tests/test_streams_gpu.py compares every device prior, simulator and proposal
draw with, so it is pinned here three ways: the Random123 known-answer vectors, the project's own
generator (elfi_b200/csrc/philox.cuh, built for the host by tests/harness/philox_harness.cpp) bit
for bit, and the CUDA toolkit's independent Philox (curand_philox4x32_x.h, host build by nvcc).
The Box-Muller normals of the replay are checked against mpmath, and the summation order of the
mixture CDF (cumsum_kernel) is emulated to show that the old order could make the table decrease
and that the current one cannot.
"""
import ctypes
import math
import os
import shutil
import subprocess

import numpy as np
import pytest
import scipy.stats as ss

import streams

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']

# Random123 kat_vectors (philox4x32_10): counter, key -> output
KAT = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
       ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
       ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
        (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _compile(cmd_prefix, src, tmp, name):
    so = str(tmp / name)
    subprocess.check_call(cmd_prefix + ['-o', so, os.path.join(HERE, 'harness', src)])
    return ctypes.CDLL(so)


@pytest.fixture(scope='module')
def harness(tmp_path_factory):
    gxx = shutil.which('g++')
    if gxx is None:
        pytest.skip('g++ not available')
    return _compile([gxx, '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared'],
                    'philox_harness.cpp', tmp_path_factory.mktemp('philox'), 'philox_harness.so')


@pytest.fixture(scope='module')
def curand_harness(tmp_path_factory):
    nvcc = shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'
    if not os.path.exists(nvcc):
        pytest.skip('nvcc not available')
    return _compile([nvcc, '-O2', '-std=c++17', '-Xcompiler', '-fPIC', '-shared'] + ARCH,
                    'curand_philox_harness.cu', tmp_path_factory.mktemp('curand'),
                    'curand_philox_harness.so')


def _seed(key):
    return key[0] | (key[1] << 32)


def _counters(n, rs):
    """Random counters and keys plus the edges: zero, all ones, row high words != 0."""
    ctr = rs.randint(0, 2 ** 32, size=(n, 4), dtype=np.uint64).astype(np.uint32)
    key = rs.randint(0, 2 ** 32, size=(n, 2), dtype=np.uint64).astype(np.uint32)
    edges = [0, 1, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFE, 0xFFFFFFFF]
    e = np.array([(a, b, c, d) for a in edges for b in edges[:3] for c in (0, 1, 0xFFFFFFFF)
                  for d in (0, streams.SALT_GM_RVS, 0xFFFFFFFF)], dtype=np.uint32)
    ek = np.array([(e[i, 0] ^ e[i, 2], e[i, 1] | (i & 1) * 0xFFFFFFFF) for i in range(len(e))],
                  dtype=np.uint32)
    return np.concatenate([ctr, e]), np.concatenate([key, ek])


def _replay(ctr, key):
    seed = key[:, 0].astype(np.uint64) | (key[:, 1].astype(np.uint64) << np.uint64(32))
    out = streams.philox4x32_10(ctr[:, 0], ctr[:, 1], ctr[:, 2], ctr[:, 3], seed)
    return np.stack(out, axis=1).astype(np.uint32), seed


@pytest.mark.parametrize('ctr,key,expect', KAT)
def test_replay_known_answers(ctr, key, expect):
    got = streams.philox4x32_10(*ctr, _seed(key))
    assert tuple(int(w) for w in got) == expect


def test_replay_vectorised_over_rows_matches_scalar():
    rows = np.array([0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 40 + 3], dtype=np.uint64)
    vec = streams.philox4x32_10(rows & np.uint64(0xFFFFFFFF), rows >> np.uint64(32), 5, 7, 2 ** 33 + 9)
    for i, r in enumerate(rows):
        one = streams.philox4x32_10(int(r) & 0xFFFFFFFF, int(r) >> 32, 5, 7, 2 ** 33 + 9)
        assert tuple(int(w[i]) for w in vec) == tuple(int(w) for w in one)


def test_project_generator_equals_replay(harness):
    rs = np.random.RandomState(5)
    ctr, key = _counters(100000, rs)
    want, seed = _replay(ctr, key)
    got = np.empty_like(ctr)
    harness.harness_philox(_ptr(np.ascontiguousarray(ctr)), _ptr(seed), ctypes.c_int64(len(ctr)),
                           _ptr(got))
    assert np.array_equal(got, want)
    for c, k, expect in KAT:
        one = np.array([c], dtype=np.uint32)
        s = np.array([_seed(k)], dtype=np.uint64)
        out = np.empty((1, 4), dtype=np.uint32)
        harness.harness_philox(_ptr(one), _ptr(s), ctypes.c_int64(1), _ptr(out))
        assert tuple(int(w) for w in out[0]) == expect


def test_project_u01_equals_replay(harness):
    rs = np.random.RandomState(6)
    a = np.concatenate([rs.randint(0, 2 ** 32, 100000, dtype=np.uint64),
                        [0, 0, 0xFFFFFFFF, 0xFFFFFFFF, 0, 0]]).astype(np.uint32)
    b = np.concatenate([rs.randint(0, 2 ** 32, 100000, dtype=np.uint64),
                        [0, 0x7FF, 0xFFFFFFFF, 0, 0xFFF, 0x800]]).astype(np.uint32)
    got = np.empty(a.size)
    harness.harness_u01(_ptr(a), _ptr(b), ctypes.c_int64(a.size), _ptr(got))
    want = streams.u01(a, b)
    assert np.array_equal(got.view(np.int64), want.view(np.int64))
    # the mapping itself: 53 bits, (0, 1], smallest 2^-53, largest exactly 1
    assert want[-6] == 2.0 ** -53 and want[-5] == 2.0 ** -53 and want[-4] == 1.0
    assert want[-2] == 2.0 ** -52 and want[-1] == 2.0 ** -52
    assert want.min() > 0.0 and want.max() <= 1.0
    v = (want * 2.0 ** 53 - 1).astype(np.uint64)
    assert np.array_equal(v >> np.uint64(21), a.astype(np.uint64) & np.uint64(0xFFFFFFFF))
    assert np.array_equal(v & np.uint64(0x1FFFFF), b.astype(np.uint64) >> np.uint64(11))


def test_replay_equals_toolkit_philox(curand_harness):
    rs = np.random.RandomState(7)
    ctr, key = _counters(100000, rs)
    want, _ = _replay(ctr, key)
    got = np.empty_like(ctr)
    curand_harness.harness_curand_philox(_ptr(np.ascontiguousarray(ctr)), _ptr(np.ascontiguousarray(key)),
                                         ctypes.c_int64(len(ctr)), _ptr(got))
    assert np.array_equal(got, want)


def test_replay_normals_against_mpmath():
    """Box-Muller of the replay (exact argument reduction of sinpi / cospi) within 1e-15 of the
    correctly rounded normals; the device tolerance of 1e-14 max(1, rad) rests on this."""
    mpmath = pytest.importorskip('mpmath')
    rs = np.random.RandomState(8)
    words = [rs.randint(0, 2 ** 32, 3000, dtype=np.uint64) for _ in range(4)]
    # edges of the angle: v in {1/4, 1/2, 3/4, 1} and next to them
    words[2][:8] = [0x40000000, 0x3FFFFFFF, 0x80000000, 0x7FFFFFFF, 0xC0000000, 0xBFFFFFFF,
                    0xFFFFFFFF, 0]
    words[3][:8] = [0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF,
                    0xFFFFFFFF, 0]
    n0, n1, rad = streams.normal2(words)
    u, v = streams.u01(words[0], words[1]), streams.u01(words[2], words[3])
    mpmath.mp.prec = 120
    for i in range(u.size):
        r = mpmath.sqrt(-2 * mpmath.log(mpmath.mpf(float(u[i]))))
        t = 2 * mpmath.mpf(float(v[i]))
        z0, z1 = float(r * mpmath.cospi(t)), float(r * mpmath.sinpi(t))
        tol = 1e-15 * max(1.0, float(r))
        assert abs(n0[i] - z0) <= tol and abs(n1[i] - z1) <= tol, (i, n0[i], z0, n1[i], z1)
    assert abs(rad[0] - float(mpmath.sqrt(-2 * mpmath.log(mpmath.mpf(float(u[0])))))) <= 1e-15 * rad[0]


def _zero_heavy_weights(rs, n):
    w = rs.rand(n) ** 8
    w[rs.rand(n) < 0.3] = 0.0
    return w


def test_old_cdf_order_can_decrease_new_order_cannot():
    """The summation order of the former cumsum_kernel (warp shuffle scan per 1024-tile) makes
    the CDF table decrease after zero weights; the current kernel's order (sequential per thread,
    scanned bases, running maximum) is nondecreasing for the same weights."""
    rs = np.random.RandomState(9)
    dips_old = dips_new = 0
    for _ in range(200):
        w = _zero_heavy_weights(rs, 3000)
        old = streams.gm_cdf_warp_scan(w, w.size)
        new = streams.gm_cdf(w)
        dips_old += int(np.sum(np.diff(old) < 0))
        dips_new += int(np.sum(np.diff(new) < 0))
        np.testing.assert_allclose(new, np.cumsum(w), rtol=1e-12, atol=0)
        assert abs(new[-1] - math.fsum(w)) <= 1e-13 * math.fsum(w)
        # a zero weight adds nothing: its entry equals its predecessor's, so the first-index
        # search can never stop on it
        z = np.flatnonzero(w[1:] == 0) + 1
        assert np.array_equal(new[z], new[z - 1])
    assert dips_old > 100
    assert dips_new == 0


@pytest.mark.parametrize('n', [1, 7, 8191, 8192, 8193, 100000])
def test_new_cdf_order_shapes(n):
    rs = np.random.RandomState(n)
    for w in (_zero_heavy_weights(rs, n), rs.rand(n) * 10.0 ** rs.randint(-12, 12, n), None):
        got = streams.gm_cdf(w, n)
        ref = np.cumsum(np.ones(n) if w is None else w)
        np.testing.assert_allclose(got, ref, rtol=1e-12, atol=0)
        assert np.all(np.diff(got) >= 0)
        if w is None:
            assert np.array_equal(got, ref)             # integers: exact


def test_replay_search_and_zero_weight_components():
    """The replay's binary search is np.searchsorted(side='left') on a sorted table, and with the
    current table a zero-weight component is never chosen."""
    rs = np.random.RandomState(10)
    w = _zero_heavy_weights(rs, 5000)
    w[0] = w[-1] = 0.0
    cumw = streams.gm_cdf(w)
    u = rs.rand(200000) * cumw[-1]
    c = streams._first_ge(cumw, u)
    assert np.array_equal(c, np.searchsorted(cumw, u, side='left'))
    assert np.all(w[c] > 0)


@pytest.mark.parametrize('a,b', [(0.01, 10.0), (3.0, 8.0), (6.0, 9.0), (9.0, 12.0), (-12.0, -9.0),
                                 (-1.0, 2.0)])
def test_replayed_truncnorm_prior_follows_scipy(a, b):
    """The inverse-CDF formula the device prior uses (mirrored in the upper tail) draws from
    scipy.stats.truncnorm(a, b) also far out in either tail."""
    mu, sigma = streams.prior_gauss(100000, 3, [0.0, 1.0, a, b])
    assert np.all((sigma >= a) & (sigma <= b))
    assert np.unique(sigma).size > 99000
    assert ss.kstest(sigma, ss.truncnorm(a, b).cdf).pvalue > 1e-3
    assert ss.kstest(mu, 'uniform').pvalue > 1e-3
    mpmath = pytest.importorskip('mpmath')
    mpmath.mp.dps = 60
    mass = streams.gauss_prior_constants([0.0, 1.0, a, b])[4]
    ref = float(mpmath.ncdf(b) - mpmath.ncdf(a))
    assert abs(mass - ref) <= 1e-13 * ref, (mass, ref)
