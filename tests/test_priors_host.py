"""CPU checks of the stock-prior arithmetic (elfi_b200/csrc/priors.cuh, built for the host by
tests/harness/priors_harness.cpp), of its NumPy replay (tests/prior_replay.py), of
DeviceModelPrior's model validation, and of the samplers driving DeviceModelPrior on the CPU test
double."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import scipy.stats as ss

import device_prior_cases as cases
import prior_replay as pr
import streams

HERE = os.path.dirname(os.path.abspath(__file__))


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.fixture(scope='module')
def harness(tmp_path_factory):
    gxx = shutil.which('g++')
    if gxx is None:
        pytest.skip('g++ not available')
    so = str(tmp_path_factory.mktemp('priors') / 'priors_harness.so')
    subprocess.check_call([gxx, '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-o', so,
                           os.path.join(HERE, 'harness', 'priors_harness.cpp')])
    return ctypes.CDLL(so)


def _spec(kind, params):
    from elfi_b200.priors import prior_spec
    return np.asarray(prior_spec(kind, params), dtype=np.float64)


def _host_logpdf(harness, specs, x):
    specs = np.ascontiguousarray(np.atleast_2d(specs), dtype=np.float64)
    x = np.ascontiguousarray(x.reshape(len(x), -1), dtype=np.float64)
    out = np.empty(len(x))
    why = ctypes.create_string_buffer(200)
    rc = harness.harness_prior_logpdf(_ptr(specs), ctypes.c_int64(len(specs)), _ptr(x),
                                      ctypes.c_int64(len(x)), _ptr(out), why, ctypes.c_int64(200))
    return rc, out, why.value.decode()


def edge_points(spec, rs, n=2000):
    """Random points around the support, its edges exactly, one ulp beyond them, far outside."""
    lo, hi = pr.support(spec)
    kind, shapes, loc, scale = pr.unpack(spec)
    flo = lo if np.isfinite(lo) else loc - 10 * scale
    fhi = hi if np.isfinite(hi) else loc + 10 * scale
    w = fhi - flo
    x = rs.uniform(flo - 0.2 * w, fhi + 0.2 * w, n)
    extra = [flo + 1e-300 + 0.0 * w, -1e300, 1e300, np.inf, -np.inf]
    for e in (lo, hi):
        if np.isfinite(e):
            extra += [e, np.nextafter(e, np.inf), np.nextafter(e, -np.inf)]
    return np.concatenate([x, extra])


def _agree(got, ref, what):
    assert np.array_equal(np.isposinf(got), np.isposinf(ref)), what
    assert np.array_equal(np.isneginf(got), np.isneginf(ref)), what
    assert np.array_equal(np.isnan(got), np.isnan(ref)), what
    fin = np.isfinite(ref)
    np.testing.assert_allclose(got[fin], ref[fin], rtol=1e-13, atol=1e-13, err_msg=what)


@pytest.mark.parametrize('case', cases.KIND_CASES, ids=cases.case_id)
def test_logpdf_matches_scipy(harness, case):
    """Per-kind log density vs scipy.stats: rtol 1e-13 inside the support, the same +-inf on its
    edges, one ulp beyond them and far outside, NaN for NaN."""
    spec = _spec(*case)
    x = np.concatenate([edge_points(spec, np.random.RandomState(1)), [np.nan]])
    rc, got, why = _host_logpdf(harness, spec, x)
    assert rc == 0, why
    _agree(got, pr.scipy_logpdf(spec, x), str(case))


def test_joint_logpdf_is_the_sum_of_scipy_terms(harness):
    specs = np.array([_spec(*c) for c in cases.KIND_CASES[:16]])
    rs = np.random.RandomState(2)
    x = np.column_stack([edge_points(s, rs, 300)[:300] for s in specs])
    x[:50] = np.column_stack([frozen_draws(c, 50, rs) for c in cases.KIND_CASES[:16]])
    rc, got, why = _host_logpdf(harness, specs, x)
    assert rc == 0, why
    ref = pr.joint_logpdf(specs, x)
    assert np.isfinite(ref[:50]).all()
    _agree(got, ref, 'joint')


def frozen_draws(case, n, rs):
    return cases.frozen(*case).rvs(size=n, random_state=rs)


@pytest.mark.parametrize('spec,index,message', [
    ([[0, 0, 1, 0, 0], [1, 0, 0, 0, 0]], 1, 'scale'),
    ([[2, 3, 3, 0, 1]], 0, 'truncnorm needs a < b'),
    ([[0, 0, 1, 0, 0], [0, 0, 1, 0, 0], [4, 0, 0, 1, 0]], 2, 'gamma needs'),
    ([[5, 1, -1, 0, 1]], 0, 'beta needs'),
    ([[6, 0, 1, 0, 0]], 0, 'unknown kind'),
    ([[0, 0, np.inf, 0, 0]], 0, 'scale')])
def test_invalid_parameters_are_refused(harness, spec, index, message):
    """The host constants builder refuses bad parameters and names them; ops refuses the same
    table with a ValueError before any library call."""
    from elfi_b200 import ops
    spec = np.asarray(spec, dtype=np.float64)
    rc, _, why = _host_logpdf(harness, spec, np.zeros((1, len(spec))))
    assert rc == -1 - index and message in why, (rc, why)
    with pytest.raises(ValueError, match='prior parameter {}: .*{}'.format(index, message)):
        ops._prior_table(spec)


def test_truncnorm_log_mass_in_the_tails(harness):
    mpmath = pytest.importorskip('mpmath')
    mpmath.mp.dps = 60
    for a, b in [(9.0, 12.0), (-12.0, -9.0), (-1.0, 2.0), (0.0, 5.0), (-1e-3, 1e-3), (30.0, 31.0)]:
        out = np.empty(13)
        why = ctypes.create_string_buffer(200)
        assert harness.harness_prior_entry(_ptr(np.array([2.0, a, b, 0.0, 1.0])), _ptr(out), why,
                                           ctypes.c_int64(200)) == 0
        ref = float(mpmath.log(mpmath.ncdf(b) - mpmath.ncdf(a)))
        assert abs(out[1] - ref) <= 1e-13 * abs(ref) + 1e-15, (a, b, out[1], ref)


@pytest.mark.parametrize('shape', [0.3, 1.0, 2.5, 0.5, 5.0])
def test_marsaglia_tsang_decisions_match_replay(harness, shape):
    """The acceptance test of priors.cuh against the replay's: the same decision and v wherever
    the decision is not within 1e-12 of the bound."""
    d, c, _ = pr.gamma_constants(shape)
    rs = np.random.RandomState(3)
    z = np.concatenate([rs.randn(200000), [-1.0 / c, -1.0 / c - 1e-9, -1.0 / c + 1e-9, 0.0, 8.0]])
    u = np.concatenate([rs.rand(200000), [0.5, 0.5, 0.5, 1.0, 1.0]])
    u[u == 0] = 1.0
    acc = np.empty(z.size, dtype=np.int32)
    v = np.empty(z.size)
    margin = np.empty(z.size)
    harness.harness_mt_accept(ctypes.c_double(d), ctypes.c_double(c), _ptr(z), _ptr(u),
                              ctypes.c_int64(z.size), _ptr(acc), _ptr(v), _ptr(margin))
    racc, rv, rmargin = pr.mt_trial(d, c, z, u)
    sure = rmargin > 1e-12
    assert (~sure).sum() <= 5
    assert np.array_equal(acc[sure].astype(bool), racc[sure])
    np.testing.assert_allclose(v[racc], rv[racc], rtol=1e-15)
    assert 0.9 < racc.mean() < 1.0                    # Marsaglia-Tsang accepts most trials


# ------------------------------------------------------------------------------ replay
@pytest.mark.parametrize('case', cases.KIND_CASES, ids=cases.case_id)
def test_replayed_prior_draws_follow_scipy(case):
    """The stream formulas of prior_rvs_kernel (as replayed) draw from scipy.stats.<kind>: KS
    p > 1e-3 at 1e5 draws; gamma / beta need a second trial on some rows and never the bound."""
    spec = _spec(*case)
    x, err, trial, margin = pr.prior_rvs(spec, 100000, 2 ** 32 + 17, 2 ** 32 - 50000)
    assert ss.kstest(x, cases.frozen(*case).cdf).pvalue > 1e-3
    assert np.isfinite(pr.scipy_logpdf(spec, x)).all() or case[0] in ('gamma', 'beta')
    lo, hi = pr.support(spec)
    assert np.all((x >= lo) & (x <= hi))
    if case[0] in ('gamma', 'beta'):
        assert trial.min() >= 0 and (trial >= 1).any()


def test_replayed_proposals_equal_the_p4_replay():
    """For p <= 4 with supports 0 and 2 the wide replay draws what oracle/streams.gm_rvs draws."""
    rs = np.random.RandomState(4)
    for p in (1, 2, 3, 4):
        means = rs.uniform(-1, 1, (50, p))
        L = np.linalg.cholesky(np.eye(p) * 0.1 + 0.01)
        cumw = streams.gm_cdf(rs.rand(50))
        box = (np.full(p, -0.9), np.full(p, 0.9))
        for support, bx in ((0, None), (2, box)):
            a = pr.gm_rvs(means, L, cumw, 3000, 2 ** 32 + 1, 7, support, bx)
            b = streams.gm_rvs(means, L, cumw, 3000, 2 ** 32 + 1, 7, support, bx)
            for u, v in zip(a, b):
                assert np.array_equal(u, v)


# ------------------------------------------------------------------------------ DeviceModelPrior
def _model(*priors):
    from elfi_b200 import model as em
    m = em.new_model()
    for name, args in priors:
        em.Prior(*args, model=m, name=name)
    return m


@pytest.mark.parametrize('args,kind,spec', [
    (('uniform', 0, 10), 'uniform', [0, 0, 10, 0, 0]),
    (('unif', 0, 10), 'uniform', [0, 0, 10, 0, 0]),
    ((ss.uniform,), 'uniform', [0, 0, 1, 0, 0]),
    (('norm', 50, 7), 'norm', [1, 50, 7, 0, 0]),
    (('normal',), 'norm', [1, 0, 1, 0, 0]),
    (('Normal', 2), 'norm', [1, 2, 1, 0, 0]),
    ((ss.expon, np.e, 2), 'expon', [3, np.e, 2, 0, 0]),
    (('exponential',), 'expon', [3, 0, 1, 0, 0]),
    (('truncnorm', 0, 5), 'truncnorm', [2, 0, 5, 0, 1]),
    ((ss.truncnorm, 0, 5, 1, 2), 'truncnorm', [2, 0, 5, 1, 2]),
    (('gamma', 2), 'gamma', [4, 2, 0, 1, 0]),
    ((ss.gamma, 2, 0, 0.5), 'gamma', [4, 2, 0, 0.5, 0]),
    (('beta', 2, 3), 'beta', [5, 2, 3, 0, 1]),
    ((ss.beta, 0.5, 0.5, -1, 2), 'beta', [5, 0.5, 0.5, -1, 2]),
    (('uniform', np.float32(1.5), np.int64(2)), 'uniform', [0, 1.5, 2, 0, 0])])
def test_device_model_prior_accepts_stock_priors(args, kind, spec):
    import elfi_b200 as elfi
    dp = elfi.DeviceModelPrior(_model(('a', args)))
    assert dp.parameter_names == ['a'] and dp.kinds == [kind]
    np.testing.assert_array_equal(dp.specs, [spec])


def test_device_model_prior_orders_parameters_like_the_model():
    import elfi_b200 as elfi
    m = cases.six_model()
    dp = elfi.DeviceModelPrior(m)
    assert dp.parameter_names == m.parameter_names == cases.SIX_NAMES
    assert dp.kinds == [k for k, _ in cases.SIX_PRIORS]
    # the device copy keeps names, parents and observed data; the original is untouched
    assert dp.model.nodes == m.nodes and dp.model.observed.keys() == m.observed.keys()
    for n in m.parameter_names:
        assert dp.model.get_parents(n) == m.get_parents(n)
        assert m[n].distribution is getattr(ss, dp.kinds[cases.SIX_NAMES.index(n)])
        assert dp.model[n].distribution.kind == dp.kinds[cases.SIX_NAMES.index(n)]


def test_device_copy_keeps_the_host_model_prior():
    """The twins' pdf / logpdf are scipy's, so ModelPrior of the device copy equals the original's."""
    import elfi_b200 as elfi
    m = cases.six_model()
    dp = elfi.DeviceModelPrior(m)
    rs = np.random.RandomState(5)
    x = np.column_stack([cases.frozen(*c).rvs(size=200, random_state=rs) for c in cases.SIX_PRIORS])
    x[:20] -= 1.5
    with np.errstate(all='ignore'):
        a = elfi.ModelPrior(m).logpdf(x)
        b = elfi.ModelPrior(dp.model).logpdf(x)
    assert np.array_equal(a, b)


def test_device_model_prior_rejects_what_it_cannot_run():
    import elfi_b200 as elfi
    from elfi_b200 import model as em
    from elfi_b200.examples import ma2
    with pytest.raises(ValueError, match="prior 't1': custom distribution CustomPrior1"):
        elfi.DeviceModelPrior(ma2.get_model(seed_obs=1))
    m = em.new_model()
    t1 = em.Prior('uniform', 0, 10, model=m, name='t1')
    em.Prior('uniform', t1, 10, model=m, name='t2')                  # mg1's t2 = U(t1, 10)
    with pytest.raises(ValueError, match="prior 't2': parameter 0 depends on node 't1'"):
        elfi.DeviceModelPrior(m)
    with pytest.raises(ValueError, match="prior 'v' is a vector prior"):
        elfi.DeviceModelPrior(_vector_model())
    for dist in ('lognorm', 'halfnorm', ss.lognorm, 'poisson'):
        with pytest.raises(ValueError, match="is not supported on the device \\(supported: uniform, "
                                             "norm, truncnorm, expon, gamma, beta\\)"):
            elfi.DeviceModelPrior(_model(('x', (dist, 1.0))))
    with pytest.raises(ValueError, match="prior 'x': truncnorm takes from 2 to 4"):
        elfi.DeviceModelPrior(_model(('x', ('truncnorm', 1.0))))
    with pytest.raises(ValueError, match="prior 'x': uniform takes at most 2"):
        elfi.DeviceModelPrior(_model(('x', ('uniform', 0, 1, 2))))
    with pytest.raises(ValueError, match="prior 'x': .*scale"):
        elfi.DeviceModelPrior(_model(('x', ('norm', 0, -1))))
    with pytest.raises(ValueError, match="prior 'x': gamma needs"):
        elfi.DeviceModelPrior(_model(('x', ('gamma', 0))))
    with pytest.raises(ValueError, match="prior 'x': parameter 0 is not a real scalar"):
        elfi.DeviceModelPrior(_model(('x', ('norm', np.zeros(2)))))
    with pytest.raises(ValueError, match='at most 16'):
        elfi.DeviceModelPrior(_model(*[('p{:02d}'.format(i), ('uniform',)) for i in range(17)]))


def _vector_model():
    from elfi_b200 import model as em
    m = em.new_model()
    em.Prior('norm', 0, 1, size=3, model=m, name='v')
    return m


# ------------------------------------------------------------------------------ samplers (double)
@pytest.fixture
def prior_double(cpu_double, monkeypatch):
    import abi_double
    import priors_double
    abi_double.install(monkeypatch, priors_double.TABLE)
    return cpu_double


def test_ops_on_the_double(prior_double):
    from elfi_b200 import ops
    specs = np.array([_spec(*c) for c in cases.SIX_PRIORS])
    x = ops.prior_rvs(specs[4], 5000, seed=3).cpu().numpy()
    assert ss.kstest(x, cases.frozen(*cases.SIX_PRIORS[4]).cdf).pvalue > 1e-3
    theta = np.column_stack([cases.frozen(*c).rvs(size=100, random_state=np.random.RandomState(i))
                             for i, c in enumerate(cases.SIX_PRIORS)])
    np.testing.assert_array_equal(ops.prior_logpdf(theta, specs).cpu().numpy(),
                                  pr.joint_logpdf(specs, theta))
    y = ops.gm_rvs(theta, np.eye(6) * 0.5, None, 4000, seed=1, support=3, prior=specs).cpu().numpy()
    assert np.isfinite(pr.joint_logpdf(specs, y)).all()
    with pytest.raises(ValueError, match='prior parameter 2'):
        ops.prior_logpdf(theta[:, :3], [[0, 0, 1, 0, 0], [0, 0, 1, 0, 0], [2, 1, 1, 0, 1]])


def _posterior_check(res, ref, what):
    """Posterior means within 4 Monte-Carlo standard errors of each other (ESS-based)."""
    a, b = res.sample_means_array, ref.sample_means_array
    se = []
    for r in (res, ref):
        w = r.weights if r.weights is not None else np.ones(r.n_samples)
        ess = w.sum() ** 2 / (w ** 2).sum()
        se.append(r.samples_array.std(axis=0) / np.sqrt(ess))
    tol = 4 * np.sqrt(se[0] ** 2 + se[1] ** 2)
    assert np.all(np.abs(a - b) <= tol), (what, a, b, tol)


def test_smc_with_device_model_prior_on_the_double(prior_double):
    import elfi_b200 as elfi
    m = cases.six_model()
    dp = elfi.DeviceModelPrior(m)
    res = elfi.SMC(dp.model['d'], batch_size=5000, seed=4, device_proposal=dp).sample(
        1000, quantiles=[0.2, 0.3], bar=False)
    assert 'elfi_b200_prior_rvs_f64' in prior_double.CALLS
    assert 'elfi_b200_prior_logpdf_f64' in prior_double.CALLS
    assert np.isfinite(pr.joint_logpdf(dp.specs, res.samples_array)).all()
    ref = elfi.SMC(m['d'], batch_size=5000, seed=4).sample(1000, quantiles=[0.2, 0.3], bar=False)
    _posterior_check(res, ref, 'SMC')


def test_adaptive_threshold_smc_with_device_model_prior_on_the_double(prior_double):
    import elfi_b200 as elfi
    m = cases.six_model()
    dp = elfi.DeviceModelPrior(m)
    res = elfi.AdaptiveThresholdSMC(dp.model['d'], batch_size=4000, seed=4,
                                    device_proposal=dp).sample(500, max_iter=3, bar=False)
    assert 2 <= len(res.populations) <= 3
    assert np.isfinite(pr.joint_logpdf(dp.specs, res.samples_array)).all()
    obs = dp.model.observed['sim'][0]
    assert np.all(np.abs(res.sample_means_array - obs) < 0.6), (res.sample_means_array, obs)
