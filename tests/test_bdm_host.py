"""CPU checks of the birth-death-mutation (BDM) example.

* elfi_b200/csrc/bdm.cuh built for the host (tests/harness/bdm_harness.cpp), driven by the
  reference executable's generator (std::mt19937 and uniform_real_distribution<double>), against
  that executable as oracle/ref_bins.mk builds it (oracle/_ref/bdm): byte for byte, at several seeds,
  the four law points, N = 1 and N = 1024;
* the header fed the Philox uniforms against tests/bdm_replay.py, row for row, and its summaries
  against NumPy and the reference's T1 / T2 (tests/golden/gen_golden_bdm.py) bit for bit;
* the host path of elfi_b200.examples.bdm (the executable through tools.external_operation)
  against the reference's draws and Rejection sample;
* tools.external_operation;
* the Python layer (validation, the throughput-mode graph) on the CPU test double extended by
  tests/bdm_double.py.
"""
import ctypes
import os
import shutil
import subprocess
import warnings

import numpy as np
import pytest

import bdm_replay
import streams
from conftest import ROOT, load_golden

HERE = os.path.dirname(os.path.abspath(__file__))
EXE = os.path.join(ROOT, 'oracle', '_ref', 'bdm')
needs_exe = pytest.mark.skipif(
    not os.path.isfile(EXE),
    reason='oracle/_ref/bdm absent: ELFI_REFERENCE_ROOT=<reference checkout> make -C oracle '
           '-f ref_bins.mk')
LAW_POINTS = [(0.2, 0.0, 0.198, 20), (0.005, 0.0, 0.198, 20), (1.0, 0.3, 0.198, 20),
              (1.0, 0.1, 0.198, 473)]


@pytest.fixture(scope='module')
def harness(tmp_path_factory):
    gxx = shutil.which('g++')
    if gxx is None:
        pytest.skip('g++ not available')
    so = str(tmp_path_factory.mktemp('bdm') / 'bdm_harness.so')
    subprocess.check_call([gxx, '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-o',
                           so, os.path.join(HERE, 'harness', 'bdm_harness.cpp')])
    return ctypes.CDLL(so)


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _harness_mt(harness, P, seed):
    """The executable's stdout as the harness produces it for rows P (B, 4)."""
    P = np.ascontiguousarray(P, dtype=np.float64)
    out = np.zeros((len(P), 1024), dtype=np.uint32)
    assert harness.harness_bdm_mt(_ptr(P), ctypes.c_int64(len(P)), ctypes.c_uint32(seed),
                                  _ptr(out), ctypes.c_int64(1024)) == 0
    return ''.join(' '.join(str(v) for v in out[i, :int(P[i, 3])]) + '\n'
                   for i in range(len(P))).encode()


def _harness_rows(harness, P, N, seed, offset, max_events):
    """The header run on the kernel's Philox uniforms: (X, n_events)."""
    P = np.ascontiguousarray(P, dtype=np.float64)
    _, n_ref = bdm_replay.simulate(P, N, seed, offset, max_events)
    K = max(int(n_ref.max()), 1)
    rows = streams.rows_of(len(P), offset)
    u, v = np.empty((len(P), K)), np.empty((len(P), K))
    for k in range(K):
        u[:, k], v[:, k] = bdm_replay.uniforms(rows, np.full(len(P), k), seed)
    X = np.empty((len(P), N), dtype=np.int16)
    n = np.empty(len(P), dtype=np.int64)
    harness.harness_bdm_rows(_ptr(P), ctypes.c_int64(len(P)), ctypes.c_int32(N), _ptr(u), _ptr(v),
                             ctypes.c_int64(K), ctypes.c_int64(max_events), _ptr(X), _ptr(n))
    return X, n


def _host_summaries(x, n=20):
    from elfi_b200.examples import bdm
    with np.errstate(all='ignore'):
        return np.column_stack([bdm.T1(x), bdm.T2(x, n)])


# ---------------------------------------------------------------------------- the header
@needs_exe
@pytest.mark.parametrize('seed', [7, 1, 2 ** 32 - 1])
def test_header_matches_executable_byte_for_byte(harness, tmp_path, seed):
    P = np.array([p for p in LAW_POINTS for _ in range(60)] + [(1.3, 0.2, 0.198, 1)] * 20
                 + [(1.5, 0.1, 0.25, 1024)] * 8 + [(0.7, 0.69, 0.05, 40)] * 30)
    inp = tmp_path / 'in.txt'
    np.savetxt(inp, P, fmt='%.4f %.4f %.4f %d')
    ref = subprocess.run([EXE, str(inp), '--seed', str(seed), '--mode', '1'], check=True,
                         stdout=subprocess.PIPE).stdout
    assert _harness_mt(harness, np.loadtxt(inp), seed) == ref


def test_header_matches_replay(harness):
    P = np.array([p[:3] for p in LAW_POINTS[:3] for _ in range(100)]
                 + [(-1.0, 0, 1), (0, 0, 0), (np.nan, 0, 1), (1, np.inf, 1), (1e308, 1e308, 1e308),
                    (0, 0.5, 0)])
    for N, offset in ((20, 0), (1, 2 ** 32 - 40), (35, 5)):
        X, n = bdm_replay.simulate(P, N, 3, offset)
        Xh, nh = _harness_rows(harness, P, N, 3, offset, 2 ** 24)
        assert np.array_equal(X, Xh) and np.array_equal(n, nh), N
        assert np.all(n[-6:-1] == -1) and np.all(X[-6:-1] == -1)
        # only deaths: extinct at the first event
        assert n[-1] == 1 and np.all(X[-1] == 0)
    # capped rows, among them a lone individual that only mutates (it never ends)
    Q = np.vstack([P[:50], [(0, 0, 0.3)]])
    X, n = bdm_replay.simulate(Q, 20, 3, 0, max_events=30)
    Xh, nh = _harness_rows(harness, Q, 20, 3, 0, 30)
    assert np.array_equal(X, Xh) and np.array_equal(n, nh)
    assert n[-1] == 30 and np.all(X[-1] == -1) and np.all(X[n < 30] >= 0)


def test_header_summaries_match_numpy_and_reference(harness):
    g = load_golden('bdm_summaries')
    for name in ('extinct', 'n1', 'n473', 'n1024', 'n20'):
        x = np.ascontiguousarray(g['x_' + name])
        for key, n in (('t2_', 20), ('t2n7_', 7), ('t2n473_', 473)):
            h = _host_summaries(x, n)
            assert np.array_equal(h[:, 0], g['t1_' + name], equal_nan=True), name
            assert np.array_equal(h[:, 1], g[key + name], equal_nan=True), (name, n)
            S = np.empty((len(x), 2))
            harness.harness_bdm_summaries(_ptr(x), ctypes.c_int64(len(x)),
                                          ctypes.c_int32(x.shape[1]), ctypes.c_double(n), _ptr(S))
            assert np.array_equal(S, h, equal_nan=True), (name, n)
    assert np.isnan(g['t1_extinct'][0])
    rs = np.random.RandomState(1)
    for N in (1, 7, 8, 9, 127, 128, 129, 256, 300, 513, 1000, 1024):
        x = rs.randint(0, 30, (4, N)).astype(np.int16)
        S = np.empty((4, 2))
        harness.harness_bdm_summaries(_ptr(x), ctypes.c_int64(4), ctypes.c_int32(N),
                                      ctypes.c_double(20.0), _ptr(S))
        assert np.array_equal(S, _host_summaries(x)), N


# ---------------------------------------------------------------------------- host mode
@pytest.fixture
def with_exe(tmp_path, monkeypatch):
    if not os.path.isfile(EXE):
        pytest.skip('oracle/_ref/bdm absent: ELFI_REFERENCE_ROOT=<reference checkout> make -C '
                    'oracle -f ref_bins.mk')
    shutil.copy(EXE, tmp_path / 'bdm')
    monkeypatch.chdir(tmp_path)
    return tmp_path


def _host(v):
    return v.cpu().numpy() if hasattr(v, 'cpu') else np.asarray(v)


def test_host_draws_match_reference_golden(with_exe, cpu_double):
    from elfi_b200.examples import bdm
    g = load_golden('bdm_draws')
    m = bdm.get_model()
    assert m.name == 'bdm'
    assert np.array_equal(m.observed['BDM'], g['observed'])
    for B, s in ((1, 1), (7, 2), (300, 3)):
        out = m.generate(B, ['BDM', 'T1', 'd'], seed=s)
        for k in ('BDM', 'T1', 'd'):
            want = g['{}_B{}_s{}'.format(k, B, s)]
            got = _host(out[k])
            assert got.dtype == want.dtype and np.array_equal(got, want), (k, B, s)
    assert os.listdir(with_exe) == ['bdm']   # the batch files are removed


def test_host_rejection_matches_reference_golden(with_exe, cpu_double):
    import elfi_b200 as elfi
    from elfi_b200.examples import bdm
    g = load_golden('bdm_rejection')
    m = bdm.get_model()
    res = elfi.Rejection(m['d'], batch_size=1000, seed=1).sample(200, quantile=0.1, bar=False)
    assert res.n_sim == int(g['n_sim'])
    assert res.threshold == float(g['threshold'])
    assert np.array_equal(res.discrepancies, g['d'])
    # T1 takes few values, so many rows tie: the rows below the threshold are the same set; the
    # order within a tie, and which tied rows at the threshold are kept, follow the sort
    below = g['d'] < g['threshold']
    assert below.sum() > 100
    assert np.array_equal(np.sort(res.samples['alpha'][below]), np.sort(g['alpha'][below]))


def test_host_seed_obs_and_summaries(with_exe, cpu_double):
    from elfi_b200.examples import bdm
    m = bdm.get_model(seed_obs=3)
    y = m.observed['BDM']
    assert y.dtype == np.int16 and y.shape == (20,) and y.sum() == 20
    m2 = bdm.get_model(seed_obs=3, N=40)
    assert m2.observed['BDM'].shape == (40,) and m2.observed['BDM'].sum() == 40
    assert sorted(os.listdir(with_exe)) == ['bdm']
    x = _host(m.generate(5, ['BDM'], seed=1)['BDM'])
    assert np.array_equal(bdm.T2(x), 1 - np.sum((x / 20) ** 2, axis=1))


def test_get_model_warns_without_executable(tmp_path, monkeypatch):
    from elfi_b200.examples import bdm
    monkeypatch.chdir(tmp_path)
    with pytest.warns(RuntimeWarning, match='bdm.cpp'):
        bdm.get_model()
    (tmp_path / 'bdm').write_text('')
    with warnings.catch_warnings():
        warnings.simplefilter('error')
        bdm.get_model()


# ---------------------------------------------------------------------------- external_operation
def test_external_operation_echo_int8():
    import elfi_b200 as elfi
    assert 'external_operation' in elfi.tools.__all__
    op = elfi.tools.external_operation('echo 1 {0}', process_result='int8')
    m = elfi.new_model()
    sim = elfi.Simulator(op, elfi.Constant(123, model=m), model=m)
    out = sim.generate()
    assert out.dtype == np.int8 and np.array_equal(out, [1, 123])
    op = elfi.tools.external_operation('echo 2.5,{0}', sep=',')
    assert np.array_equal(op(4), [2.5, 4.0])


def test_external_operation_seed_and_meta():
    from elfi_b200 import tools
    from elfi_b200.model import get_sub_seed
    op = tools.external_operation('echo {seed} {batch_index} {model_name} {x}',
                                  process_result=lambda out, *a, **k: out.decode().split())
    rs = np.random.RandomState(5)
    first = rs.get_state()[1][0]
    meta = dict(model_name='m', batch_index=4, submission_index=0)
    for index in (None, 0, 3):
        kw = dict(meta, index_in_batch=index) if index is not None else dict(meta)
        out = op(random_state=rs, meta=kw, x=9)
        assert out == [str(get_sub_seed(first, index or 0)), '4', 'm', '9'], index
    # explicit keyword inputs win over meta keys of the same name
    assert op(meta=dict(meta, x=1, seed=2), x=3)[3] == '3'
    with pytest.raises(KeyError, match='seed'):
        op(x=1, meta=meta)


def test_external_operation_completed_process_and_check(tmp_path):
    from elfi_b200 import tools
    seen = []

    def handler(completed, *inputs, **kwinputs):
        seen.append((completed.returncode, inputs, kwinputs['tag']))
        return completed.stdout

    op = tools.external_operation('echo {0} {tag}', process_result=handler, stdout=False,
                                  subprocess_kwargs=dict(stdout=subprocess.PIPE))
    assert op(5, tag='t') == b'5 t\n' and seen == [(0, (5,), 't')]
    op = tools.external_operation('exit 3')
    with pytest.raises(subprocess.CalledProcessError):
        op()
    op = tools.external_operation('exit 3', subprocess_kwargs=dict(check=False))
    assert op().size == 0
    prepared = tools.external_operation(
        'cat {path}', prepare_inputs=lambda *a, **k: (a, dict(k, path=str(tmp_path / 'f'))))
    (tmp_path / 'f').write_text('7 8')
    assert np.array_equal(prepared(), [7.0, 8.0])


# ---------------------------------------------------------------------------- Python layer
@pytest.fixture
def bdm_double(cpu_double, monkeypatch):
    import bdm_double
    import priors_double
    priors_double.install(monkeypatch)
    bdm_double.install(monkeypatch)
    return cpu_double


def test_ops_validate_before_the_call(bdm_double):
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    P = np.tile([0.2, 0.0, 0.198], (3, 1))
    for N in (0, 1025, 2.5):
        with pytest.raises(ValueError, match='1 <= N <= 1024'):
            ops.sim_bdm(P, N)
    for me in (0, 2 ** 32, 1.5):
        with pytest.raises(ValueError, match='max_events'):
            ops.sim_bdm(P, 20, max_events=me)
    with pytest.raises(ValueError, match='parameter width of 2'):
        ops.sim_bdm(P[:, :2], 20)
    with pytest.raises(ValueError, match='1 <= N <= 1024'):
        ops.bdm_summaries(np.zeros((2, 1025), dtype=np.int16))
    with pytest.raises(ValueError, match='batch, N'):
        ops.bdm_summaries(dev.to_device(np.zeros((2, 3, 4))))
    assert not bdm_double.CALLS
    X, S, n = ops.sim_bdm(P, 1024)
    assert tuple(X.shape) == (3, 1024) and tuple(S.shape) == (3, 2) and tuple(n.shape) == (3,)
    X, S, n = ops.sim_bdm(P, 20, want_data=False)
    assert X is None and S is not None


def test_dispatch_host_device_and_lazy_agree(bdm_double):
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    from elfi_b200.examples import bdm
    x = load_golden('bdm_draws')['BDM_B300_s3']
    h = _host_summaries(x)
    assert np.array_equal(ops.bdm_summaries(x).cpu().numpy(), h)
    xd = dev.to_device(x.astype(np.float64))
    assert np.array_equal(bdm.T1(xd).cpu().numpy(), h[:, 0])
    assert np.array_equal(bdm.T2(xd, n=7).cpu().numpy(), _host_summaries(x, 7)[:, 1])
    lazy = bdm.bdm_device(0.2, 0, 0.198, 20, batch_size=50, random_state=np.random.RandomState(1))
    assert lazy.shape == (50, 20)
    t1, t2 = bdm.T1(lazy), bdm.T2(lazy)
    assert bdm_double.CALLS.count('elfi_b200_sim_bdm_f64') == 1
    data = lazy.materialize()
    assert data is lazy.materialize() and data.dtype == dev.torch.int16
    hd = data.cpu().numpy()
    assert np.all(hd.sum(axis=1) == 20)
    assert np.array_equal(t1.cpu().numpy(), _host_summaries(hd)[:, 0])
    assert np.array_equal(t2.cpu().numpy(), _host_summaries(hd)[:, 1])
    assert np.array_equal(bdm.T2(lazy, n=9).cpu().numpy(), _host_summaries(hd, 9)[:, 1])
    X, S, n = ops.sim_bdm(np.array([[-1.0, 0, 0.198], [0.2, 0, 0.198], [0.0, 0.0, 0.0]]), 20)
    X, S, n = X.cpu().numpy(), S.cpu().numpy(), n.cpu().numpy()
    assert np.all(X[[0, 2]] == -1) and np.isnan(S[[0, 2]]).all() and np.all(n[[0, 2]] == -1)
    assert X[1].sum() == 20 and n[1] > 0
    assert np.isnan(ops.bdm_summaries(X).cpu().numpy()[[0, 2]]).all()


def test_device_model_runs_rejection_and_smc(bdm_double):
    import elfi_b200 as elfi
    from elfi_b200.examples import bdm
    m, dp = bdm.get_device_model()
    assert m.name.startswith('bdm') and dp.parameter_names == ['alpha']
    assert np.array_equal(m.observed['BDM'], load_golden('bdm_draws')['observed'])
    assert sorted(n for n in m.nodes if not n.startswith('_')) == ['BDM', 'T1', 'alpha', 'd']
    res = elfi.Rejection(m['d'], batch_size=200, seed=1).sample(20, quantile=0.1, bar=False)
    assert res.n_samples == 20 and np.all(np.isfinite(res.discrepancies))
    a = res.samples['alpha']
    assert np.all((a >= 0.005) & (a <= 2.005))
    smc = elfi.SMC(m['d'], batch_size=100, seed=2, device_proposal=dp).sample(
        10, quantiles=[0.5, 0.5], bar=False)
    assert len(smc.populations) == 2
    m3, _ = bdm.get_device_model(seed_obs=3, N=30)
    y = m3.observed['BDM']
    assert y.shape == (30,) and y.sum() == 30
    m4, _ = bdm.get_device_model(seed_obs=3, N=30)
    assert np.array_equal(m4.observed['BDM'], y)
    assert 'elfi_b200_sim_bdm_f64' in bdm_double.CALLS
