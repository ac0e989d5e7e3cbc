"""CPU checks of the conditional priors (a loc or scale taken from another parameter of the row).

* elfi_b200/csrc/priors.cuh built for the host (tests/harness/conditional_priors_harness.cpp): the
  joint log density with sources against SciPy with per-row loc / scale, inside the support, on
  its edges and with per-row scales <= 0, NaN and inf (rtol 1e-13, exact infinities and NaNs);
  with every source -1 it is the 5-word table's density bit for bit; bad sources are refused;
* DeviceModelPrior(conditional=True) records the sources and refuses what it cannot run, and
  without the option refuses a node parent as before;
* the ops layer validates its inputs before any call.
"""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import scipy.stats as ss

import conditional_prior_replay as cr

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope='module')
def harness(tmp_path_factory):
    gxx = shutil.which('g++')
    if gxx is None:
        pytest.skip('g++ not available')
    d = tmp_path_factory.mktemp('cond_priors')
    out = {}
    for name in ('conditional_priors', 'priors'):
        so = str(d / (name + '_harness.so'))
        subprocess.check_call([gxx, '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared',
                               '-o', so, os.path.join(HERE, 'harness', name + '_harness.cpp')])
        out[name] = ctypes.CDLL(so)
    return out


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _logpdf(harness, specs7, x):
    specs7 = np.ascontiguousarray(specs7, dtype=np.float64)
    x = np.ascontiguousarray(x, dtype=np.float64)
    out = np.empty(x.shape[0])
    why = ctypes.create_string_buffer(256)
    rc = harness['conditional_priors'].harness_prior_logpdf_cond(
        _ptr(specs7), ctypes.c_int64(specs7.shape[0]), _ptr(x), ctypes.c_int64(x.shape[0]),
        _ptr(out), why, ctypes.c_int64(256))
    return rc, out, why.value.decode()


def _logpdf5(harness, specs, x):
    specs = np.ascontiguousarray(specs, dtype=np.float64)
    x = np.ascontiguousarray(x, dtype=np.float64)
    out = np.empty(x.shape[0])
    why = ctypes.create_string_buffer(256)
    rc = harness['priors'].harness_prior_logpdf(_ptr(specs), ctypes.c_int64(specs.shape[0]), _ptr(x),
                                                ctypes.c_int64(x.shape[0]), _ptr(out), why,
                                                ctypes.c_int64(256))
    assert rc == 0, why.value
    return out


def _close(got, want):
    """rtol 1e-13, infinities and NaNs at the same places."""
    assert got.shape == want.shape
    assert np.array_equal(np.isnan(got), np.isnan(want)), np.argwhere(np.isnan(got) != np.isnan(want))
    inf = np.isinf(want) | np.isinf(got)
    assert np.array_equal(got[inf], want[inf])
    f = np.isfinite(want)
    np.testing.assert_allclose(got[f], want[f], rtol=1e-13, atol=0)


# a parent column 0 (uniform U(0, 10)) and one conditional parameter of every kind in column 1
PARENT = [0, 0, 10, 0, 0, -1, -1]
CHILDREN = {
    'uniform loc': [0, 0, 10, 0, 0, 0, -1],
    'uniform scale': [0, 1, 1, 0, 0, -1, 0],
    'norm loc': [1, 0, 2, 0, 0, 0, -1],
    'norm scale': [1, 3, 1, 0, 0, -1, 0],
    'truncnorm both': [2, -1, 2, 0, 1, 0, 0],
    'expon loc': [3, 0, 1.5, 0, 0, 0, -1],
    'gamma scale': [4, 0.7, 0.5, 1, 0, -1, 0],
    'beta loc': [5, 2, 3, 0, 4, 0, -1],
    'beta scale': [5, 0.5, 0.8, -1, 1, -1, 0],
}


def _points(child, rs, n=600):
    t1 = rs.uniform(0, 10, n)
    t1[:40] = [0, 10, 1e-300, -0.0, 0.5, 2, 3, 7, np.nextafter(10, 11), np.nextafter(0, -1)] * 4
    spec = np.array(child, dtype=np.float64)
    _, shapes, loc, scale = cr.unpack(spec, np.column_stack([t1, t1]))
    draw_scale = np.where(np.asarray(scale) > 0, scale, 1.0)        # t1 <= 0 rows: any draw
    x2 = getattr(ss, ['uniform', 'norm', 'truncnorm', 'expon', 'gamma', 'beta'][int(spec[0])]).rvs(
        *shapes, loc, draw_scale, size=n, random_state=rs) if spec[0] != 2 else \
        loc + scale * rs.uniform(-1.5, 2.5, n)
    x2 = np.asarray(x2, dtype=np.float64)
    x2[40:80] = np.asarray(loc + 0 * t1)[40:80]                             # on the loc edge
    x2[80:100] = np.nextafter(np.asarray(loc + 0 * t1)[80:100], -np.inf)    # one ulp below it
    if spec[0] in (0, 5):
        hi = np.asarray(loc + scale * 1.0 + 0 * t1)
        x2[100:120] = hi[100:120]
        x2[120:140] = np.nextafter(hi[120:140], np.inf)
    x2[140:150] = [np.nan, np.inf, -np.inf, 0.0, -0.0, 1e308, -1e308, 5.0, 1e-320, -1.0]
    return np.column_stack([t1, x2])


@pytest.mark.parametrize('name', sorted(CHILDREN))
def test_logpdf_with_sources_matches_scipy(harness, name):
    rs = np.random.RandomState(sorted(CHILDREN).index(name))
    specs7 = np.array([PARENT, CHILDREN[name]], dtype=np.float64)
    x = _points(CHILDREN[name], rs)
    rc, got, why = _logpdf(harness, specs7, x)
    assert rc == 0, why
    _close(got, cr.joint_logpdf(specs7, x))
    assert np.isfinite(got).sum() > 200


def test_per_row_scale_rule_matches_scipy(harness):
    """A sourced scale <= 0 or NaN gives NaN, an infinite one -inf for uniform; a NaN loc NaN."""
    specs7 = np.array([[0, 0, 1, 0, 0, -1, 0], [1, -5, 10, 0, 0, -1, -1]], dtype=np.float64)
    scales = np.array([-1.0, -0.0, 0.0, np.nan, np.inf, -np.inf, 1e-310, 2.0])
    x = np.column_stack([np.zeros_like(scales) + 0.5, scales])
    # column 0: uniform(loc 1, scale = column 1); column 1: its own constant norm
    specs7 = np.array([[0, 1, 1, 0, 0, -1, 1], [1, 0, 10, 0, 0, -1, -1]], dtype=np.float64)
    rc, got, why = _logpdf(harness, specs7, x)
    assert rc == 0, why
    want = cr.joint_logpdf(specs7, x)
    _close(got, want)
    assert np.isnan(got[:4]).all() and np.isnan(got[5])
    # uniform loc NaN, and an infinite scale with a finite point
    specs7 = np.array([[0, 0, 1, 0, 0, 1, 2], [1, 0, 10, 0, 0, -1, -1], [0, 0, 10, 0, 0, -1, -1]],
                      dtype=np.float64)
    x = np.array([[0.5, np.nan, 1.0], [0.5, 0.0, np.inf], [3.0, 0.0, np.inf], [np.inf, 0.0, np.inf]])
    rc, got, why = _logpdf(harness, specs7, x)
    _close(got, cr.joint_logpdf(specs7, x))
    assert np.isnan(got[0]) and np.isneginf(got[1]) and np.isneginf(got[2]) and np.isnan(got[3])


def test_no_sources_is_the_five_word_table_bit_for_bit(harness):
    import device_prior_cases as cases
    from elfi_b200.priors import prior_spec
    specs = np.array([prior_spec(k, p) for k, p in cases.SIX_PRIORS])
    rs = np.random.RandomState(3)
    x = np.column_stack([cases.frozen(*c).rvs(size=500, random_state=rs) for c in cases.SIX_PRIORS])
    x[:50] += rs.normal(0, 1, (50, x.shape[1]))
    x[50:60] = np.nan
    specs7 = np.concatenate([specs, -np.ones((len(specs), 2))], axis=1)
    rc, got, why = _logpdf(harness, specs7, x)
    assert rc == 0, why
    want = _logpdf5(harness, specs, x)
    assert np.array_equal(got.view(np.int64), want.view(np.int64))


def test_bad_sources_are_refused(harness):
    x = np.zeros((1, 2))
    for src, msg in (((1, -1), 'loc source'), ((-1, 2), 'scale source'), ((0.5, -1), 'loc source'),
                     ((-2, -1), 'loc source')):
        specs7 = np.array([PARENT, [0, 0, 1, 0, 0, -1, -1]], dtype=np.float64)
        specs7[1, 5:] = src
        if src[0] == 1:                       # the parameter itself
            specs7 = np.array([[0, 0, 1, 0, 0, -1, -1], [0, 0, 1, 0, 0, 1, -1]], dtype=np.float64)
        rc, _, why = _logpdf(harness, specs7, x)
        assert rc == -2 and msg in why, (src, why)
    # a placeholder word is not validated; a shape word always is
    specs7 = np.array([PARENT, [0, np.nan, -3, 0, 0, 0, 0]], dtype=np.float64)
    assert _logpdf(harness, specs7, x)[0] == 0
    specs7 = np.array([PARENT, [4, -1, 0, 1, 0, 0, -1]], dtype=np.float64)
    rc, _, why = _logpdf(harness, specs7, x)
    assert rc == -2 and 'gamma needs' in why


# ---------------------------------------------------------------------------- DeviceModelPrior
def _model(*priors):
    from elfi_b200 import model as em
    m = em.new_model()
    for name, args in priors:
        em.Prior(*[m[a] if isinstance(a, str) and a in m.nodes else a for a in args], model=m,
                 name=name)
    return m


def test_device_model_prior_records_sources():
    import elfi_b200 as elfi
    m = _model(('a', ('uniform', 0, 10)), ('b', ('uniform', 'a', 10)), ('c', ('norm', 'a', 'b')),
               ('d', ('gamma', 2.0, 'c')), ('e', ('norm', 0, 1)))
    dp = elfi.DeviceModelPrior(m, conditional=True)
    assert dp.parameter_names == ['a', 'b', 'c', 'd', 'e']
    np.testing.assert_array_equal(dp.sources, [[-1, -1], [0, -1], [0, 1], [2, -1], [-1, -1]])
    np.testing.assert_array_equal(dp.specs[1], [0, 0, 10, 0, 0])
    np.testing.assert_array_equal(dp.specs[2], [1, 0, 1, 0, 0])
    np.testing.assert_array_equal(dp.specs[3], [4, 2, 0, 1, 0])
    from elfi_b200.examples import mg1
    dp = elfi.DeviceModelPrior(mg1.get_model(seed_obs=1), conditional=True)
    assert dp.parameter_names == ['t1', 't2', 't3']
    np.testing.assert_array_equal(dp.sources, [[-1, -1], [0, -1], [-1, -1]])
    for conditional in (False, True):
        dp = elfi.DeviceModelPrior(_model(('a', ('uniform', 0, 10)), ('b', ('norm', 1, 2))),
                                   conditional=conditional)
        np.testing.assert_array_equal(dp.sources, -np.ones((2, 2)))


def test_conditional_device_model_prior_refusals():
    """Without conditional=True a node parent is refused as before, with a pointer to the option;
    with it, a node in a shape position, a parent that is not a Prior and vector priors are
    refused, naming the node."""
    import elfi_b200 as elfi
    from elfi_b200 import model as em
    from elfi_b200.examples import mg1
    with pytest.raises(ValueError, match="prior 't2': parameter 0 depends on node 't1'.*"
                                         "conditional=True"):
        elfi.DeviceModelPrior(mg1.get_model(seed_obs=1))
    m = em.new_model()
    em.Prior('uniform', 0, 10, model=m, name='t1')
    em.Prior('gamma', m['t1'], 1, model=m, name='g')
    with pytest.raises(ValueError, match="prior 'g': its shape parameter 0 \\(a\\) depends on node "
                                         "'t1'"):
        elfi.DeviceModelPrior(m, conditional=True)
    m = em.new_model()
    em.Prior('uniform', 0, 10, model=m, name='t1')
    em.Prior('truncnorm', -1, m['t1'], model=m, name='tn')
    with pytest.raises(ValueError, match="prior 'tn': its shape parameter 1 \\(b\\)"):
        elfi.DeviceModelPrior(m, conditional=True)
    m = em.new_model()
    t1 = em.Prior('uniform', 0, 10, model=m, name='t1')
    em.Operation(np.abs, t1, model=m, name='op')
    em.Prior('norm', m['op'], 1, model=m, name='x')
    with pytest.raises(ValueError, match="prior 'x': parameter 0 depends on node 'op' \\(Operation\\)"):
        elfi.DeviceModelPrior(m, conditional=True)
    m = em.new_model()
    em.Prior('norm', 0, 1, size=3, model=m, name='v')
    em.Prior('norm', m['v'], 1, model=m, name='w')
    with pytest.raises(ValueError, match="vector prior"):
        elfi.DeviceModelPrior(m, conditional=True)
    with pytest.raises(ValueError, match="prior 't1': custom distribution CustomPrior1"):
        from elfi_b200.examples import ma2
        elfi.DeviceModelPrior(ma2.get_model(seed_obs=1), conditional=True)


# ---------------------------------------------------------------------------- ops validation
@pytest.fixture
def cond_double(cpu_double, monkeypatch):
    import abi_double
    import mg1_double
    import priors_double
    abi_double.install(monkeypatch, priors_double.TABLE, mg1_double.TABLE)
    return cpu_double


def test_ops_validate_before_the_call(cond_double):
    from elfi_b200 import ops
    specs = np.array([[0, 0, 10, 0, 0], [0, 0, 10, 0, 0]], dtype=np.float64)
    x = np.ones((3, 2))
    for src, msg in (([[-1, -1], [1, -1]], 'other than 1'), ([[-1, -1], [2, -1]], 'column'),
                     ([[-1, -1], [0.5, -1]], 'column'), ([[-1], [0]], r'\(p, 2\)')):
        with pytest.raises(ValueError, match=msg):
            ops.prior_logpdf(x, specs, np.array(src))
        with pytest.raises(ValueError, match=msg):
            ops.gm_rvs(x[:, :2], np.eye(2), None, 4, seed=1, support=4, prior=specs,
                       sources=np.array(src))
    with pytest.raises(ValueError, match='sources'):
        ops.gm_rvs(x[:, :2], np.eye(2), None, 4, seed=1, support=4, prior=specs)
    with pytest.raises(ValueError, match='loc has 2 values for 3 draws'):
        ops.prior_rvs([0, 0, 1, 0, 0], 3, seed=1, loc=np.zeros(2))
    with pytest.raises(ValueError, match='scale'):
        ops.prior_rvs([0, 0, -1, 0, 0], 3, seed=1, loc=np.zeros(3))
    assert not cond_double.CALLS
    ops.prior_rvs([0, 0, -1, 0, 0], 3, seed=1, scale=np.ones(3))    # the placeholder is not read
    assert cond_double.CALLS == ['elfi_b200_prior_rvs_cond_f64']


def test_ops_dispatch_on_the_double(cond_double):
    from elfi_b200 import ops
    specs = np.array([[0, 0, 10, 0, 0], [0, 0, 10, 0, 0]], dtype=np.float64)
    src = np.array([[-1, -1], [0, -1]])
    x = np.array([[1.0, 5.0], [1.0, 0.5], [2.0, 12.0], [2.0, 12.5]])
    lp = ops.prior_logpdf(x, specs, src).cpu().numpy()
    np.testing.assert_array_equal(np.isfinite(lp), [True, False, True, False])
    assert ops.prior_logpdf(x, specs).cpu().numpy()[1] == -np.log(100)
    t1 = ops.prior_rvs([0, 0, 10, 0, 0], 4000, seed=2)
    t2 = ops.prior_rvs([0, 0, 10, 0, 0], 4000, seed=3, loc=t1).cpu().numpy()
    d = t2 - t1.cpu().numpy()
    assert d.min() >= 0 and d.max() <= 10 and ss.kstest(d, ss.uniform(0, 10).cdf).pvalue > 1e-3
    g = ops.gm_rvs(np.array([[5.0, 6.0]]), np.eye(2) * 4, None, 3000, seed=5, support=4,
                   prior=specs, sources=src).cpu().numpy()
    assert np.isfinite(cr.joint_logpdf(np.concatenate([specs, src], axis=1), g)).all()
    assert 'elfi_b200_prior_logpdf_cond_f64' in cond_double.CALLS
    assert 'elfi_b200_prior_logpdf_f64' in cond_double.CALLS
