"""CPU checks of the scratch assay example and of elfi_b200.tools.

* the host path of elfi_b200.examples.scratch_assay against the golden fixtures of the unmodified
  reference (tests/golden/gen_golden_scratch_assay.py), bit for bit: draws (a lattice that fills,
  an empty lattice, a random reduced lattice), cell_summaries, the observed data, the weights and
  a Rejection sample; the graph names match the reference;
* tools.vectorize: the constants mask, dtype=False, automatic constants, the length check and
  meta['index_in_batch'];
* elfi_b200/csrc/scratch_assay.cuh built for the host (tests/harness/scratch_assay_harness.cpp):
  its lattices and summaries equal the NumPy replay of the streams (tests/scratch_assay_replay.py)
  bit for bit, and its law matches the reference-style host cell_sim (KS tests);
* ops rejects shapes outside its limits with ValueError, before any call.
"""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import scipy.stats as ss

import scratch_assay_replay as rp
from conftest import load_golden

HERE = os.path.dirname(os.path.abspath(__file__))
REDUCED = [8, 10, 20, 3]


@pytest.fixture(scope='module')
def harness(tmp_path_factory):
    gxx = shutil.which('g++')
    if gxx is None:
        pytest.skip('g++ not available')
    so = str(tmp_path_factory.mktemp('scratch_assay') / 'scratch_assay_harness.so')
    subprocess.check_call([gxx, '-O2', '-std=c++17', '-fPIC', '-shared', '-o', so,
                           os.path.join(HERE, 'harness', 'scratch_assay_harness.cpp')])
    return ctypes.CDLL(so)


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def run_harness(h, P, init, num_obs, interval, seed, offset=0, want_data=True):
    P = np.ascontiguousarray(P, dtype=np.float64).reshape(-1, 2)
    init = np.ascontiguousarray(np.asarray(init) != 0, dtype=np.uint8)
    B, (nrows, ncols) = P.shape[0], init.shape
    X = np.empty((B, nrows, ncols, num_obs + 1), dtype=np.uint8) if want_data else None
    S = np.empty((B, num_obs + 1))
    h.harness_scratch_assay(_ptr(P), ctypes.c_int64(B), _ptr(init), ctypes.c_int32(nrows),
                            ctypes.c_int32(ncols), ctypes.c_int32(num_obs),
                            ctypes.c_int32(interval), ctypes.c_uint64(seed),
                            ctypes.c_uint64(offset), _ptr(X) if want_data else None, _ptr(S))
    return X, S


# ---------------------------------------------------------------------------- reference goldens
def test_host_draws_match_reference_golden():
    from elfi_b200 import tools
    from elfi_b200.examples import scratch_assay as sa
    g = load_golden('scratch_assay_draws')
    init = g['obs'][0, :, :, 0]
    assert np.array_equal(sa.cell_sim(0.25, 0.002, init_arr=init,
                                      random_state=np.random.RandomState(5)), g['given'])
    vec = tools.vectorize(sa.cell_sim, constants=(2,))
    batch = vec(g['prm'][:, 0], g['prm'][:, 1], init, random_state=np.random.RandomState(6))
    assert batch.dtype == np.float64 and np.array_equal(batch, g['batch'])
    fill = sa.cell_sim(0.3, 1.0, init_arr=init, random_state=np.random.RandomState(7))
    assert np.array_equal(fill, g['fill'])
    assert np.all(fill[:, :, -1] == 1)           # the lattice filled: the full-lattice path ran
    empty = sa.cell_sim(0.5, 0.5, init_arr=np.zeros((6, 7)), random_state=np.random.RandomState(8))
    assert np.array_equal(empty, g['empty']) and not empty.any()
    reduced = sa.cell_sim(0.4, 0.05, init_params=REDUCED, random_state=np.random.RandomState(9))
    assert np.array_equal(reduced, g['reduced'])


def test_host_summaries_match_reference_golden():
    from elfi_b200.examples import scratch_assay as sa
    g = load_golden('scratch_assay_summaries')
    d = load_golden('scratch_assay_draws')
    for name, arr in (('obs', d['obs']), ('given', d['given'][None]), ('batch', d['batch']),
                      ('fill', d['fill'][None]), ('empty', d['empty'][None]),
                      ('reduced', d['reduced'][None]), ('crafted', g['crafted']),
                      ('real', g['real'])):
        assert np.array_equal(sa.cell_summaries(arr), g[name + '_sums']), name
    # boolean data gives the same values
    assert np.array_equal(sa.cell_summaries(d['batch'] != 0), g['batch_sums'])


def test_observed_weights_and_rejection_match_reference_golden(cpu_double):
    import elfi_b200 as elfi
    from elfi_b200.examples import scratch_assay as sa
    g = load_golden('scratch_assay_rejection')
    m = sa.get_model(init_params=REDUCED, seed_obs=1)
    assert np.array_equal(m.observed['sim'], g['observed'])
    assert sorted(n for n in m.nodes if not n.startswith('_')) == list(g['names'])
    assert m.parameter_names == ['pm', 'pp']
    _, _, weis = sa._observed(None, None, REDUCED, 1)
    assert np.array_equal(weis, g['weights'])
    res = elfi.Rejection(m['d'], batch_size=20, seed=3).sample(10, quantile=0.25, bar=False)
    assert res.n_sim == int(g['n_sim'])
    assert res.threshold == float(g['threshold'])
    assert np.array_equal(res.discrepancies, g['d'])
    for name in ('pm', 'pp'):
        assert np.array_equal(res.samples[name], g['out_' + name]), name


def test_default_observed_data_match_reference_golden():
    from elfi_b200.examples import scratch_assay as sa
    g = load_golden('scratch_assay_draws')
    obs, first, weis = sa._observed(None, None, None, 4)
    assert np.array_equal(obs, g['obs']) and np.array_equal(first, g['obs'][0, :, :, 0])
    assert weis.shape == (145,) and weis[-1] == 1 / np.sum(first) ** 2


# ---------------------------------------------------------------------------- tools.vectorize
def test_vectorize_constants_and_automatic_constants():
    from elfi_b200 import tools
    seen = []

    def op(a, b, c, random_state=None):
        seen.append((a, b, c))
        return a + b + np.sum(c)
    vec = tools.vectorize(op, constants=(2,))
    out = vec(np.array([1.0, 2.0]), 10.0, np.array([5.0, 6.0, 7.0]))
    assert np.array_equal(out, [29.0, 30.0])
    assert [s[1] for s in seen] == [10.0, 10.0]                 # a scalar is passed whole
    assert all(np.array_equal(s[2], [5.0, 6.0, 7.0]) for s in seen)
    # a list is not an array either; a 0-d array is passed whole
    seen.clear()
    out = tools.vectorize(op)(np.array([1.0, 2.0, 3.0]), np.array(1.0), [1, 2])
    assert np.array_equal(out, [5.0, 6.0, 7.0]) and all(s[2] == [1, 2] for s in seen)
    # without batched inputs the batch has one row
    assert np.array_equal(tools.vectorize(op)(1.0, 2.0, 3.0), [6.0])


def test_vectorize_dtype_false_length_check_and_meta():
    from elfi_b200 import tools

    def op(a, meta=None, batch_size=None):
        return np.arange(int(a)), dict(meta)
    outs = tools.vectorize(op, dtype=False)(np.array([1, 3]), meta={'model_name': 'x'})
    assert outs.dtype == object and outs.shape == (2,)
    assert np.array_equal(outs[1][0], [0, 1, 2])
    assert [o[1]['index_in_batch'] for o in outs] == [0, 1]
    with pytest.raises(ValueError, match='does not match'):
        tools.vectorize(lambda a, b: a)(np.ones(3), np.ones(4))
    with pytest.raises(ValueError, match='does not match'):
        tools.vectorize(lambda a: a)(np.ones(3), batch_size=2)
    out = tools.vectorize(lambda a: np.array([a, a]), dtype=np.float32)(np.array([1, 2]))
    assert out.dtype == np.float32 and out.shape == (2, 2)


def test_vectorize_consumes_one_random_state_row_after_row():
    from elfi_b200 import tools

    def op(a, random_state=None):
        return random_state.uniform(size=2) + a
    out = tools.vectorize(op)(np.array([0.0, 10.0]), random_state=np.random.RandomState(3))
    want = np.random.RandomState(3).uniform(size=4).reshape(2, 2) + [[0.0], [10.0]]
    assert np.array_equal(out, want)
    import elfi_b200
    assert elfi_b200.tools.vectorize is tools.vectorize


# ---------------------------------------------------------------------------- header on the host
DEFAULT_PARAMS = np.array([[0.25, 0.002], [0.0, 0.0], [0.0, 1.0], [1.0, 0.0], [1.0, 1.0],
                           [1.5, -0.5], [np.nan, 0.3], [0.3, np.nan], [0.9, 0.5], [0.05, 0.02]])


def test_header_equals_replay_at_the_reduced_lattice(harness):
    rs = np.random.RandomState(0)
    init = np.zeros((8, 10))
    init.reshape(-1)[rs.permutation(30)[:20]] = 1
    P = np.vstack([DEFAULT_PARAMS, rs.uniform(0, 1, (10, 2))])
    for offset in (0, 2 ** 32 - 7):
        X, S = run_harness(harness, P, init, 144, 2, seed=11, offset=offset)
        Xr, Sr = rp.sim(P, init, 144, 2, seed=11, offset=offset)
        assert np.array_equal(X, Xr) and np.array_equal(S, Sr), offset
        assert np.array_equal(S, rp.summaries(X))
    # pm, pp outside [0, 1] and NaN behave as 1 or 0: no NaN row
    assert np.isfinite(S).all()
    assert np.array_equal(S[1, :-1], np.zeros(144)) and S[1, -1] == 20      # nothing happens


def test_header_equals_replay_at_the_default_size(harness):
    g = load_golden('scratch_assay_draws')
    init = g['obs'][0, :, :, 0]
    P = DEFAULT_PARAMS[[0, 2, 4, 6, 8]]
    X, S = run_harness(harness, P, init, 144, 2, seed=5, offset=2 ** 32 - 2)
    Xr, Sr = rp.sim(P, init, 144, 2, seed=5, offset=2 ** 32 - 2)
    assert np.array_equal(X, Xr) and np.array_equal(S, Sr)
    # pp = 1 fills the lattice; after that every frame is full and the mismatches are 0
    full = np.flatnonzero(S[1, :-1] == 0)
    assert S[1, -1] == 972 and full.size > 0 and np.all(X[1, :, :, full[0] + 1:] == 1)
    # the summaries without the frames are the same
    _, S2 = run_harness(harness, P, init, 144, 2, seed=5, offset=2 ** 32 - 2, want_data=False)
    assert np.array_equal(S2, S)


def test_header_full_and_empty_lattices(harness):
    P = np.array([[0.5, 0.5], [1.0, 1.0]])
    for init, count in ((np.ones((5, 6)), 30), (np.zeros((5, 6)), 0)):
        X, S = run_harness(harness, P, init, 12, 3, seed=1)
        assert np.all(X == init[None, :, :, None]) and np.all(S[:, :-1] == 0)
        assert np.all(S[:, -1] == count)
    # one free site: pp = 1 fills it, after which nothing changes
    init = np.ones((4, 4))
    init[2, 3] = 0
    X, S = run_harness(harness, np.array([[0.0, 1.0]]), init, 5, 1, seed=2)
    Xr, Sr = rp.sim([[0.0, 1.0]], init, 5, 1, seed=2)
    assert np.array_equal(X, Xr) and np.array_equal(S, Sr)
    assert S[0, :-1].sum() == 1 and S[0, -1] == 16


def test_header_rows_across_2_32_and_observation_spacing(harness):
    init = np.zeros((6, 9))
    init[:2, ::2] = 1
    P = np.tile([[0.6, 0.1]], (6, 1))
    for interval, num_obs in ((1, 20), (3, 7), (5, 0)):
        X, S = run_harness(harness, P, init, num_obs, interval, seed=3, offset=2 ** 32 - 3)
        Xr, Sr = rp.sim(P, init, num_obs, interval, seed=3, offset=2 ** 32 - 3)
        assert np.array_equal(X, Xr) and np.array_equal(S, Sr), interval
    # row i of a launch at offset o is row 0 of a launch at offset o + i
    _, one = run_harness(harness, P[:1], init, 20, 1, seed=3, offset=2 ** 32 + 1)
    _, many = run_harness(harness, P, init, 20, 1, seed=3, offset=2 ** 32 - 3)
    assert np.array_equal(one[0], many[4])


@pytest.mark.parametrize('pm_pp', [(0.25, 0.002), (0.6, 0.05), (0.1, 0.2)])
def test_header_law_matches_reference_style_cell_sim(harness, pm_pp):
    """KS tests of the final count and the total mismatch at the reduced lattice: the header's law
    against the reference-style host cell_sim, from the same initial lattice."""
    from elfi_b200.examples import scratch_assay as sa
    init = sa._random_init(*REDUCED, random_state=np.random.RandomState(1))
    n = 300
    rs = np.random.RandomState(2)
    host = np.array([sa.cell_summaries(sa.cell_sim(*pm_pp, init_arr=init, random_state=rs)[None])[0]
                     for _ in range(n)])
    _, S = run_harness(harness, np.tile(pm_pp, (4 * n, 1)), init, 144, 2, seed=9, want_data=False)
    for name, a, b in (('count', host[:, -1], S[:, -1]),
                       ('mismatch', host[:, :-1].sum(1), S[:, :-1].sum(1))):
        p = ss.ks_2samp(a, b).pvalue
        assert p > 1e-4, (pm_pp, name, p)


# ---------------------------------------------------------------------------- ops limits
def test_ops_reject_shapes_outside_the_limits(cpu_double):
    from elfi_b200 import ops
    from elfi_b200.examples import scratch_assay as sa
    ok = np.zeros((8, 10))
    with pytest.raises(ValueError, match='4096 sites'):
        ops.sim_scratch_assay(np.ones((2, 2)) * 0.5, np.zeros((65, 64)))
    with pytest.raises(ValueError, match='2-d'):
        ops.sim_scratch_assay(np.ones((2, 2)) * 0.5, np.zeros(10))
    with pytest.raises(ValueError, match='0s and 1s'):
        ops.sim_scratch_assay(np.ones((2, 2)) * 0.5, np.full((3, 3), 2.0))
    with pytest.raises(ValueError, match='2\\^31'):
        ops.sim_scratch_assay(np.ones((2, 2)) * 0.5, ok, obs_period=2 ** 31, tau=1)
    with pytest.raises(ValueError, match='obs_interval'):
        ops.sim_scratch_assay(np.ones((2, 2)) * 0.5, ok, obs_interval=1 / 48)
    with pytest.raises(ValueError, match='2 parameters'):
        ops.sim_scratch_assay(np.ones((2, 3)), ok)
    with pytest.raises(ValueError, match='n_frames'):
        ops.scratch_assay_summaries(np.zeros((2, 3, 4, 0)))
    with pytest.raises(ValueError, match='batch, nrows'):
        ops.scratch_assay_summaries(np.zeros((2, 3, 4)))
    with pytest.raises(ValueError, match='4096 sites'), np.errstate(divide='ignore'):
        sa.get_device_model(init_arr=np.zeros((70, 70)))          # no cells: the weights are inf
    assert 'elfi_b200_sim_scratch_assay_f64' not in cpu_double.CALLS
