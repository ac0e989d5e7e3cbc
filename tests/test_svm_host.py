"""CPU checks of the alpha-stable stochastic volatility example.

* the host path of elfi_b200.examples.stochastic_volatility_model against the golden fixtures of
  the unmodified reference (tests/golden/gen_golden_svm.py), bit for bit: draws (x_0 included),
  kurt / skew and a Rejection sample; the graph names and Constant nodes match the reference; the
  host path raises where the reference raises;
* elfi_b200/csrc/stable.cuh and svm.cuh built for the host (tests/harness/svm_harness.cpp): the
  stable draw of all three branches against a NumPy restatement of SciPy within the bound of
  tests/svm_replay.py, the S0 shift and the AR(1) log-volatility exactly, kurt / skew equal to
  NumPy's for every n in 2..512;
* the Python layer (validation, dispatch, the throughput-mode graph with its Constants) and the
  samplers on the CPU test double extended by tests/svm_double.py.
"""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import scipy.stats as ss

import svm_replay as sr
from conftest import load_golden

HERE = os.path.dirname(os.path.abspath(__file__))
FIXED = dict(kappa=1, eta=0, mu=0, phi=0.95, sigma=0.2)


@pytest.fixture(scope='module')
def harness(tmp_path_factory):
    gxx = shutil.which('g++')
    if gxx is None:
        pytest.skip('g++ not available')
    so = str(tmp_path_factory.mktemp('svm') / 'svm_harness.so')
    subprocess.check_call([gxx, '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-o', so,
                           os.path.join(HERE, 'harness', 'svm_harness.cpp')])
    return ctypes.CDLL(so)


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _same_bits(a, b):
    """Equal values, NaN where NaN, and the same sign of every zero."""
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True) and \
        np.array_equal(np.signbit(a[a == 0]), np.signbit(b[a == 0]))


# ---------------------------------------------------------------------------- reference goldens
def test_host_draws_match_reference_golden():
    from elfi_b200.examples import stochastic_volatility_model as svm
    g = load_golden('svm_draws')
    y1 = svm.alpha_stochastic_volatility_model(1.2, 0.5, **FIXED, batch_size=1,
                                               random_state=np.random.RandomState(1))
    assert _same_bits(y1, g['y1'])
    prm = g['prm']
    yb = svm.alpha_stochastic_volatility_model(prm[:, 0], prm[:, 1], **FIXED, batch_size=len(prm),
                                               random_state=np.random.RandomState(2))
    assert _same_bits(yb, g['yb'])
    yx = svm.alpha_stochastic_volatility_model(prm[:, 0], prm[:, 1], **FIXED, n_obs=20, x_0=0.3,
                                               batch_size=len(prm),
                                               random_state=np.random.RandomState(3))
    assert _same_bits(yx, g['yx'])
    # the corners include alpha == 1 exactly and beta = -0.0
    assert np.any(prm[:, 0] == 1.0) and np.any((prm[:, 1] == 0) & np.signbit(prm[:, 1]))


def test_host_summaries_match_reference_golden():
    from elfi_b200.examples import stochastic_volatility_model as svm
    g = load_golden('svm_summaries')
    d = load_golden('svm_draws')
    with np.errstate(all='ignore'):
        for name in ('y1', 'yb', 'yx'):
            assert _same_bits(svm.kurt(d[name]), g[name + '_kurt']), name
            assert _same_bits(svm.skew(d[name]), g[name + '_skew']), name
        for name in ('crafted', 'n2'):
            assert _same_bits(svm.kurt(g[name]), g[name + '_kurt']), name
            assert _same_bits(svm.skew(g[name]), g[name + '_skew']), name
    # the crafted rows reach NaN (0 / 0, NaN rows) and inf (q75 == q25)
    assert np.isnan(g['crafted_kurt']).any() and np.isinf(g['crafted_kurt']).any()


def test_rejection_matches_reference_golden(cpu_double):
    import elfi_b200 as elfi
    from elfi_b200.examples import stochastic_volatility_model as svm
    g = load_golden('svm_rejection')
    m = svm.get_model(seed_obs=1)
    assert _same_bits(m.observed['a_svm'], g['observed'])
    res = elfi.Rejection(m['d'], batch_size=100, seed=3).sample(20, quantile=0.1, bar=False)
    assert res.n_sim == int(g['n_sim'])
    assert res.threshold == float(g['threshold'])
    assert np.array_equal(res.discrepancies, g['d'])
    for name in ('alpha', 'beta'):
        assert np.array_equal(res.samples[name], g['out_' + name]), name


def test_graph_names_and_constants_match_the_reference():
    import elfi_b200 as elfi
    from elfi_b200.examples import stochastic_volatility_model as svm
    g = load_golden('svm_rejection')
    m = svm.get_model(seed_obs=0)
    assert sorted(n for n in m.nodes if not n.startswith('_')) == list(g['names'])
    assert m.parameter_names == ['alpha', 'beta']
    assert m.get_parents('a_svm') == ['alpha', 'beta', 'kappa', 'eta', 'mu', 'phi', 'sigma']
    for name, value in FIXED.items():
        assert m.record(name).cls is elfi.Constant and m.record(name).constant == value


def test_host_path_raises_where_the_reference_raises():
    from elfi_b200.examples import stochastic_volatility_model as svm
    bad = [dict(alpha=0.0, beta=0.5), dict(alpha=2.5, beta=0.5), dict(alpha=1.2, beta=1.5),
           dict(alpha=np.nan, beta=0.5), dict(alpha=1.2, beta=np.nan), dict(kappa=-1.0),
           dict(sigma=-0.2), dict(phi=np.nan)]
    for kw in bad:
        args = dict(alpha=1.2, beta=0.5, **FIXED)
        args.update(kw)
        with pytest.raises(ValueError):
            with np.errstate(all='ignore'):
                svm.alpha_stochastic_volatility_model(**args, n_obs=5,
                                                      random_state=np.random.RandomState(0))


# ---------------------------------------------------------------------------- headers on the host
def _stable_cases(rs, n):
    alpha = rs.uniform(0.5, 2.0, n)
    beta = rs.uniform(-1, 1, n)
    kappa = rs.uniform(0.1, 3.0, n)
    eta = rs.uniform(-2, 2, n)
    k = n // 12
    alpha[:k], alpha[k:2 * k], alpha[2 * k:3 * k] = 1.0, 2.0, 0.5
    beta[3 * k:4 * k], beta[4 * k:5 * k] = 0.0, -0.0
    beta[5 * k:6 * k], beta[6 * k:7 * k] = 1.0, -1.0
    beta[:k:3], beta[1:k:3] = 1.0, -0.0                  # alpha == 1 with beta = +-1 and -0.0
    kappa[7 * k:8 * k] = 0.0
    kappa[8 * k:9 * k] = 1.0
    kappa[:k:5] = 0.0                                     # alpha == 1, kappa == 0: NaN
    return alpha, beta, kappa, eta


@pytest.mark.parametrize('s0', [True, False])
def test_stable_draw_matches_scipy_formula(harness, s0):
    """stable.cuh's draw against the NumPy restatement of SciPy (glibc and NumPy may differ by an
    ulp in sin / cos / tan / arctan / pow / log), within svm_replay.stable's bound."""
    rs = np.random.RandomState(4)
    n = 24000
    alpha, beta, kappa, eta = _stable_cases(rs, n)
    u, v = rs.uniform(0, 1, n), 1.0 - rs.uniform(0, 1, n)
    out = np.empty(n)
    harness.harness_svm_stable(_ptr(alpha), _ptr(beta), _ptr(kappa), _ptr(eta), _ptr(u), _ptr(v),
                               ctypes.c_int64(n), ctypes.c_int32(int(s0)), _ptr(out))
    want, err, cond = sr.stable(alpha, beta, kappa, eta, u, v, s0=s0)
    assert np.array_equal(np.isnan(out), np.isnan(want))
    fin = np.isfinite(want)
    bad = fin & ~(np.abs(out - want) <= err)
    assert not bad.any(), np.argwhere(bad)[:5]
    assert np.isnan(out[(alpha == 1) & (kappa == 0)]).all()
    # kappa == 0 off alpha == 1: zero shocks, shifted to eta
    z = (alpha != 1) & (kappa == 0)
    assert np.array_equal(out[z], eta[z] - 0.0 * beta[z] * np.tan(np.pi * alpha[z] / 2))
    assert fin.mean() > 0.95
    print('largest condition number of the denominator and numerator sums: %.3g' % cond.max())


def test_stable_draw_follows_scipy(harness):
    """The three branches against scipy.stats.levy_stable itself, fed the same uniforms through a
    RandomState stand-in, S0 set on the frozen distribution's instance as the reference does."""
    rs = np.random.RandomState(8)
    for alpha, beta in ((1.0, 0.7), (1.0, 0.0), (1.4, 0.0), (1.4, -0.0), (0.7, 1.0), (2.0, -0.3),
                        (1.2, 0.5)):
        n = 500
        u, v = rs.uniform(0, 1, n), 1.0 - rs.uniform(0, 1, n)

        class Given(np.random.RandomState):
            def uniform(self, low=0.0, high=1.0, size=None):
                return u.reshape(size)

            def standard_exponential(self, size=None):
                return -np.log(v).reshape(size)

        dist = ss.levy_stable(alpha=alpha, beta=beta, loc=0.3, scale=1.7)
        dist.dist.parameterization = 'S0'
        dist.random_state = Given()
        with np.errstate(all='ignore'):
            want = dist.rvs(size=n)
        out = np.empty(n)
        full = [np.full(n, c) for c in (alpha, beta, 1.7, 0.3)]
        harness.harness_svm_stable(*(_ptr(a) for a in full), _ptr(u), _ptr(v), ctypes.c_int64(n),
                                   ctypes.c_int32(1), _ptr(out))
        _, err, _ = sr.stable(*full, u, v)
        ok = np.abs(out - want) <= err
        assert ok[np.isfinite(want)].all(), (alpha, beta)


def test_s0_shift_and_log_volatility_are_exact(harness):
    """With u = 0.5 (TH = 0) and W = 1 the draw is exact arithmetic up to tan(pi alpha / 2): the S0
    shift is checked through it.  The AR(1) from given normals equals the reference's norm.rvs
    arithmetic bit for bit, NaN rows where it raises."""
    rs = np.random.RandomState(5)
    B, n = 200, 40
    P = np.column_stack([rs.uniform(0.5, 2, B), rs.uniform(-1, 1, B), rs.uniform(0, 2, B),
                         rs.uniform(-1, 1, B), rs.uniform(-1, 1, B), rs.uniform(-1.2, 1.2, B),
                         rs.uniform(0, 1, B)])
    P[:8, 5] = [0.95, 1.0, -1.0, 0.999995, 0.0, 2.0, np.nan, 0.5]
    P[8:12, 6] = [0.0, -0.1, np.inf, np.nan]
    P[12:14, 0] = [0.0, 2.5]
    P[14:16, 1] = [1.5, np.nan]
    P[16, 2] = -1.0
    Z = rs.standard_normal((B, n))
    X = np.empty((B, n))
    ok = np.empty(B, dtype=np.int32)
    harness.harness_svm_logvol(_ptr(P), _ptr(Z), ctypes.c_int64(B), ctypes.c_int32(n), _ptr(X),
                               _ptr(ok))

    class GivenNormals(np.random.RandomState):
        def __init__(self, z):
            super().__init__(0)
            self.z, self.t = z, 0

        def standard_normal(self, size=None):
            self.t += 1
            return self.z[self.t - 1:self.t].reshape(size)

    from elfi_b200.examples import stochastic_volatility_model as svm
    for b in range(B):
        mu, phi, sigma = P[b, 4:7]
        try:
            with np.errstate(all='ignore'):
                want = svm.log_vol(mu, phi, sigma, n, random_state=GivenNormals(Z[b]))[:, 0]
            raised = False
        except ValueError:
            raised = True
        stable_ok = 0 < P[b, 0] <= 2 and -1 <= P[b, 1] <= 1 and P[b, 2] >= 0
        assert bool(ok[b]) == (not raised and stable_ok), b
        if not raised:
            assert _same_bits(X[b], want), b
    assert not ok[6] and not ok[9] and not ok[11] and ok[8] and ok[10]
    # the S0 shift: the S0 draw is the S1 draw minus it, bit for bit
    alpha = np.array([1.3, 0.7, 1.9, 1.0, 1.0])
    beta = np.array([0.5, -1.0, 1.0, 0.5, -0.0])
    kappa = np.array([1.0, 2.0, 0.5, 2.0, 3.0])
    eta = np.array([0.25, -1.0, 0.0, 0.5, 1.0])
    u, v = np.full(5, 0.5), np.full(5, np.exp(-1.0))
    s1, s0 = np.empty(5), np.empty(5)
    for s, flag in ((s1, 0), (s0, 1)):
        harness.harness_svm_stable(_ptr(alpha), _ptr(beta), _ptr(kappa), _ptr(eta), _ptr(u),
                                   _ptr(v), ctypes.c_int64(5), ctypes.c_int32(flag), _ptr(s))
    shift = np.where(alpha == 1, beta * 2 * kappa * np.log(kappa) / np.pi,
                     kappa * beta * np.tan(np.pi * alpha / 2.0))
    assert _same_bits(s0, s1 - shift)


def test_summaries_equal_numpy_for_every_n(harness):
    from elfi_b200.examples import stochastic_volatility_model as svm
    rs = np.random.RandomState(3)
    for n in range(2, 513):
        x = rs.standard_cauchy((6, n))
        x[1] = np.round(x[1])
        x[2, rs.randint(n)] = np.inf
        x[3, rs.randint(n)] = -np.inf
        x[4, rs.randint(n)] = np.nan
        x[5, :] = rs.choice([0.5, 1.0], n)
        xs = np.sort(x, axis=1)
        S = np.empty((6, 2))
        harness.harness_svm_summaries(_ptr(np.ascontiguousarray(xs)), ctypes.c_int64(6),
                                      ctypes.c_int32(n), _ptr(S))
        with np.errstate(all='ignore'):
            assert _same_bits(S[:, 0], svm.kurt(x)), n
            assert _same_bits(S[:, 1], svm.skew(x)), n


# ---------------------------------------------------------------------------- Python layer
@pytest.fixture
def svm_double(cpu_double, monkeypatch):
    import abi_double
    import priors_double
    import svm_double
    abi_double.install(monkeypatch, priors_double.TABLE, svm_double.TABLE)
    return cpu_double


def test_ops_validate_before_the_call(svm_double):
    from elfi_b200 import ops
    from elfi_b200.examples import stochastic_volatility_model as svm
    with pytest.raises(ValueError, match='observations'):
        ops.sim_svm(np.ones((2, 7)), n_obs=1)
    with pytest.raises(ValueError, match='observations'):
        ops.sim_svm(np.ones((2, 7)), n_obs=513)
    with pytest.raises(ValueError, match='7 parameters'):
        ops.sim_svm(np.ones((2, 6)))
    with pytest.raises(ValueError, match='x_0'):
        svm.svm_device(1.2, 0.5, 1, 0, 0, 0.95, 0.2, x_0=0.1, batch_size=3)
    with pytest.raises(ValueError, match='observations'):
        svm.get_device_model(n_obs=600)
    assert not svm_double.CALLS


def test_dispatch_host_device_and_lazy_agree(svm_double):
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    from elfi_b200.examples import stochastic_volatility_model as svm
    rs = np.random.RandomState(0)
    full = rs.standard_cauchy((6, 41))
    full[0, 3] = np.nan
    full[1, 1:31] = 1.0
    y = full[:, 1:]
    with np.errstate(all='ignore'):
        for src in (dev.to_device(y), dev.to_device(full)[:, 1:]):
            assert _same_bits(svm.kurt(src).cpu().numpy(), svm.kurt(y))
            assert _same_bits(svm.skew(src).cpu().numpy(), svm.skew(y))
        lazy = svm.svm_device(1.2, 0.5, 1, 0, 0, 0.95, 0.2, n_obs=30, batch_size=5,
                              random_state=np.random.RandomState(1))
        data = lazy.materialize().cpu().numpy()
        assert data.shape == (5, 30) and lazy.shape == (5, 30)
        assert _same_bits(svm.kurt(lazy).cpu().numpy(), svm.kurt(data))
        assert _same_bits(svm.skew(lazy).cpu().numpy(), svm.skew(data))
    Y, S = ops.sim_svm([[1.2, 0.5, 1, 0, 0, 0.95, 0.2], [2.5, 0.5, 1, 0, 0, 0.95, 0.2],
                        [1.2, 0.5, 1, 0, 0, np.nan, 0.2]], n_obs=8, want_data=True)
    Y, S = Y.cpu().numpy(), S.cpu().numpy()
    assert np.isfinite(Y[0]).all() and np.isnan(Y[1:]).all() and np.isnan(S[1:]).all()


def test_device_model_runs_rejection_and_smc(svm_double):
    import elfi_b200 as elfi
    from elfi_b200.examples import stochastic_volatility_model as svm
    m, dp = svm.get_device_model(seed_obs=3)
    assert dp.parameter_names == ['alpha', 'beta']
    host = svm.get_model(seed_obs=3)
    assert _same_bits(m.observed['a_svm'], host.observed['a_svm'])
    assert m.get_parents('a_svm') == host.get_parents('a_svm')

    # the Constants reach the simulator as the values the reference's loader passes
    from elfi_b200 import model as em
    seen = []

    def spy(*args, **kw):
        seen.append(args[2:7])
        return svm.svm_device(*args, **kw)
    svm._graph(em.new_model(), spy, host.observed['a_svm'])['kurt'].generate(10)
    assert seen == [(1, 0, 0, 0.95, 0.2)]

    def in_support(s):
        return np.all((s['alpha'] >= 0.5) & (s['alpha'] <= 2) & (s['beta'] >= -1) &
                      (s['beta'] <= 1))
    res = elfi.Rejection(m['d'], batch_size=500, seed=1).sample(50, quantile=0.1, bar=False)
    assert res.n_samples == 50 and in_support(res.samples)
    smc = elfi.SMC(m['d'], batch_size=500, seed=2, device_proposal=dp).sample(
        50, quantiles=[0.5, 0.5], bar=False)
    assert len(smc.populations) == 2 and in_support(smc.samples)
    m['d'].become(elfi.AdaptiveDistance(m['kurt'], m['skew']))
    ad = elfi.AdaptiveDistanceSMC(m['d'], batch_size=500, seed=3, device_proposal=dp).sample(
        50, rounds=2, quantile=0.5, bar=False)
    assert len(ad.populations) == 2 and in_support(ad.samples)
    assert 'elfi_b200_sim_svm_f64' in svm_double.CALLS
