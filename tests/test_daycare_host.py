"""CPU checks of the day care example.

* the host path of elfi_b200.examples.daycare against the golden fixtures of the unmodified
  reference (tests/golden/gen_golden_daycare.py), bit for bit: draws, summaries, distances,
  Rejection;
* elfi_b200/csrc/daycare.cuh built for the host (tests/harness/daycare_harness.cpp): the exact
  numerators of E_s, the hazards and total against the reference's formula, the selection law, the
  summaries and the distance against NumPy, and whole DCCs against the NumPy replay of the kernel
  (tests/daycare_replay.py) fed the same Philox draws;
* the Python layer (validation, dispatch, the throughput-mode graph) and the samplers on the CPU
  test double extended by tests/daycare_double.py.
"""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import load_golden

HERE = os.path.dirname(os.path.abspath(__file__))
SMALL = dict(n_dcc=5, n_ind=12, n_strains=6, n_obs=9, time_end=2.0,
             freq_strains_commun=np.array([0.05, 0.1, 0.2, 0.02, 0.3, 0.15]))


@pytest.fixture(scope='module')
def harness(tmp_path_factory):
    gxx = shutil.which('g++')
    if gxx is None:
        pytest.skip('g++ not available')
    so = str(tmp_path_factory.mktemp('dc') / 'daycare_harness.so')
    subprocess.check_call([gxx, '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-o',
                           so, os.path.join(HERE, 'harness', 'daycare_harness.cpp')])
    lib = ctypes.CDLL(so)
    lib.harness_dc_total.restype = ctypes.c_double
    return lib


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _summ(x):
    from elfi_b200.examples import daycare as dc
    return [dc.ss_shannon(x), dc.ss_strains(x), dc.ss_prevalence(x), dc.ss_prevalence_multi(x)]


def _masks(state):
    """uint64 strain masks of a (..., n_strains) bool state."""
    w = np.uint64(1) << np.arange(state.shape[-1], dtype=np.uint64)
    return (state.astype(np.uint64) * w).sum(axis=-1).astype(np.uint64)


# ---------------------------------------------------------------------------- reference goldens
def test_host_draws_match_reference_golden():
    from elfi_b200.examples import daycare as dc
    g = load_golden('daycare_draws')
    x = dc.daycare(3.6, 0.6, 0.1, random_state=np.random.RandomState(1))
    assert x.dtype == np.bool_ and np.array_equal(x, g['truth1'])
    assert np.array_equal(dc.daycare(3.6, 0.6, 0.1, batch_size=2,
                                     random_state=np.random.RandomState(2)), g['truth2'])
    P = g['mixed_prm']
    assert np.array_equal(dc.daycare(*P.T, batch_size=len(P), random_state=np.random.RandomState(3),
                                     **SMALL), g['mixed'])
    assert np.array_equal(dc.daycare(*P[4], random_state=np.random.RandomState(4), **SMALL),
                          g['small1'])


def test_host_summaries_and_distance_match_reference_golden():
    from elfi_b200.examples import daycare as dc
    g = load_golden('daycare_summaries')
    draws = load_golden('daycare_draws')
    for name in ('truth1', 'truth2', 'mixed', 'small1'):
        for j, s in enumerate(_summ(draws[name])):
            assert np.array_equal(s, g[name][j]), (name, j)
    for name in ('zeros', 'diag', 'ones'):
        for j, s in enumerate(_summ(g['x_' + name])):
            assert np.array_equal(s, g[name][j]), (name, j)
    gd = load_golden('daycare_distance')
    obs, sim = _summ(draws['truth1']), _summ(draws['truth2'])
    assert np.array_equal(dc.distance(*sim, observed=obs), gd['d_truth_b2'])
    assert np.array_equal(dc.distance(*[v[:1] for v in sim], observed=obs), gd['d_truth_b1'])
    obs_s = list(gd['obs_small'])
    assert np.array_equal(dc.distance(*gd['sim_small'], observed=obs_s), gd['d_small'])
    obs0 = [np.zeros_like(obs_s[0])] + obs_s[1:]
    assert np.array_equal(dc.distance(*gd['sim_small'], observed=obs0), gd['d_small_obs0'])
    d_nan = dc.distance(*gd['sim_nan'], observed=obs_s)
    assert np.array_equal(d_nan, gd['d_nan'], equal_nan=True) and np.isnan(d_nan[1])


def test_rejection_matches_reference_golden(cpu_double):
    import elfi_b200 as elfi
    from elfi_b200.examples import daycare as dc
    g = load_golden('daycare_rejection')
    m = dc.get_model(seed_obs=7, time_end=0.05)
    assert np.array_equal(m.observed['DCC'], g['observed'])
    res = elfi.Rejection(m['d'], batch_size=10, seed=3).sample(10, quantile=0.5, bar=False)
    assert res.n_sim == int(g['n_sim'])
    assert res.threshold == float(g['threshold'])
    assert np.array_equal(res.discrepancies, g['d'])
    for name in ('t1', 't2', 't3'):
        assert np.array_equal(res.samples[name], g['out_' + name]), name
    assert sorted(n for n in m.nodes if not n.startswith('_')) == sorted(
        ['t1', 't2', 't3', 'DCC', 'Shannon', 'n_strains', 'prevalence', 'multi', 'd', 'logd'])


# ---------------------------------------------------------------------------- the header on the host
def _reference_hazards(state, t1, t2, t3, f):
    """The hazards of daycare.py:100-118 for one DCC state (n_ind, n_strains)."""
    s = state[None, None]
    n_ind = state.shape[0]
    with np.errstate(divide='ignore', invalid='ignore'):
        adjust = np.nan_to_num(s / np.sum(s, axis=3, keepdims=True))
        prob = np.sum(adjust, axis=2, keepdims=True)
    hz = t1 * (np.tile(prob, (1, 1, n_ind, 1)) - adjust) * (1. / (n_ind - 1)) + 1e-9 + t2 * f
    hz = np.where(np.any(s, axis=3, keepdims=True), t3 * hz, hz)
    hz[s] = 1.
    return hz[0, 0], prob[0, 0, 0]


def _random_states(rs, n, n_ind, n_strains):
    for k in range(n):
        p = [0.0, 0.05, 0.3, 0.9][k % 4]
        st = rs.uniform(size=(n_ind, n_strains)) < p
        if k % 5 == 1:
            st[:] = False
        yield st


def test_header_hazards_match_reference_formula(harness):
    rs = np.random.RandomState(1)
    for n_ind, n_strains in ((53, 33), (12, 6), (64, 40), (2, 1)):
        L = 1
        for k in range(2, n_strains + 1):
            L = L * k // np.gcd(L, k)
        f = rs.uniform(0, 0.3, n_strains)
        for st in _random_states(rs, 12, n_ind, n_strains):
            for prm in ([3.6, 0.6, 0.1], [11.0, 2.0, 1.0], [0.0, 0.0, 0.0], [5.0, 0.0, 0.7]):
                h = np.empty(n_strains)
                num = np.empty(n_strains, dtype=np.int64)
                H = harness.harness_dc_total(_ptr(_masks(st)), n_ind, n_strains,
                                             _ptr(np.array(prm)), _ptr(f), _ptr(h), _ptr(num))
                n_i = st.sum(axis=1)
                want_num = [sum(L // n_i[i] for i in range(n_ind) if st[i, s])
                            for s in range(n_strains)]
                assert list(num) == want_num
                hz, E = _reference_hazards(st, *prm, f)
                # the reference sums n_ind rounded terms 1 / n_i; num / L is rounded once
                assert np.allclose(num / float(L), E, rtol=1e-14, atol=0)
                free = ~st.any(axis=1)
                if free.any():
                    np.testing.assert_allclose(h, hz[np.argmax(free)], rtol=1e-14, atol=0)
                np.testing.assert_allclose(H, hz.sum(), rtol=1e-13)


def test_header_selection_follows_the_hazards(harness):
    """On a fine grid of uniforms each transition is picked with its hazard's share of the total,
    and never one of zero hazard."""
    rs = np.random.RandomState(2)
    n_ind, n_strains = 12, 6
    f = np.array([0.05, 0.1, 0.2, 0.02, 0.3, 0.15])
    n = 400000
    x = (np.arange(n) + 0.5) / n
    for st in _random_states(rs, 8, n_ind, n_strains):
        for prm in ([3.6, 0.6, 0.1], [11.0, 2.0, 1.0], [3.6, 0.6, 0.0], [0.0, 0.0, 0.5]):
            cell = np.empty(n, dtype=np.int64)
            harness.harness_dc_pick(_ptr(_masks(st)), n_ind, n_strains, _ptr(np.array(prm)),
                                    _ptr(f), _ptr(x), ctypes.c_int64(n), _ptr(cell))
            hz, _ = _reference_hazards(st, *prm, f)
            share = np.bincount(cell, minlength=hz.size) / n
            want = (hz / hz.sum()).ravel()
            assert np.all(want[np.unique(cell)] > 0)
            assert np.abs(share - want).max() < 3.0 / n + 1e-9, prm


def test_header_refuses_unbounded_rows(harness):
    """dc_row_ok (and the replay's restatement of it): rows with t1, t2 or t3 negative, NaN or
    infinite, or whose hazards could give 2^32 - 1 transitions by time_end, do not run."""
    import daycare_replay as rp
    inf, nan = np.inf, np.nan
    P = np.array([[3.6, 0.6, 0.1], [11.0, 2.0, 1.0], [0.0, 0.0, 0.0], [inf, 0.6, 0.1],
                  [3.6, inf, 0.1], [3.6, 0.6, inf], [-inf, 0.6, 0.1], [nan, 0.6, 0.1],
                  [3.6, -1e-300, 0.1], [1e300, 0.6, 0.1], [3.6, 1e300, 0.1], [3.6, 0.6, 1e300],
                  [3e5, 0.0, 1.0], [1e5, 0.0, 1.0], [1e7, 0.0, 0.0]])
    # bound time_end n_ind n_strains c: 5.2e9 for t1 = 3e5, 1.7e9 for t1 = 1e5 (the limit is 2^32)
    want = [1, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 0]
    ok = np.empty(len(P), dtype=np.int32)
    harness.harness_dc_row_ok(_ptr(P), ctypes.c_int64(len(P)), ctypes.c_double(0.1), 53, 33,
                              ctypes.c_double(10.0), _ptr(ok))
    assert list(ok) == want
    assert list(rp.row_ok(P, np.full(33, 0.1), 53, 33, 10.0)) == [bool(v) for v in want]


def test_header_has_no_transition_without_a_positive_weight(harness):
    """Where no strain has a positive weight (parameters that dc_row_ok refuses: an infinite t1 or
    t3 makes every weight NaN, negative frequencies make them negative), dc_pick returns no
    transition and dc_step a NaN time, leaving the state alone."""
    n_ind, n_strains = 12, 6
    f = np.full(n_strains, 0.1)
    x = np.array([0.0, 0.3, 0.999])
    for prm, ff in (([np.inf, 0.6, 0.1], f), ([3.6, 0.6, np.inf], f), ([3.6, 0.6, 0.1], -f),
                    ([3.6, np.inf, 0.1], np.zeros(n_strains))):
        masks = np.zeros(n_ind, dtype=np.uint64)
        cell = np.empty(3, dtype=np.int64)
        harness.harness_dc_pick(_ptr(masks), n_ind, n_strains, _ptr(np.array(prm)), _ptr(ff),
                                _ptr(x), ctypes.c_int64(3), _ptr(cell))
        assert (cell == -1).all(), prm
        dt = np.empty(3)
        num = np.empty(n_strains, dtype=np.int64)
        harness.harness_dc_run(_ptr(masks), n_ind, n_strains, _ptr(np.array(prm)), _ptr(ff),
                               _ptr(np.ones(3)), _ptr(x), ctypes.c_int64(3), _ptr(dt), _ptr(num))
        assert np.isnan(dt).all() and not masks.any() and not num.any(), prm


def test_header_summaries_and_distance_match_numpy(harness):
    from elfi_b200.examples import daycare as dc
    rs = np.random.RandomState(3)
    g = load_golden('daycare_summaries')
    datas = [g['x_zeros'], g['x_diag'], g['x_ones'], load_golden('daycare_draws')['truth2']]
    for n_obs, n_strains in ((1, 1), (9, 6), (36, 33), (64, 64), (5, 8), (20, 17)):
        for p in (0.0, 0.05, 0.5):
            datas.append(rs.uniform(size=(3, 4, n_obs, n_strains)) < p)
    for x in datas:
        B, n_dcc, n_obs, n_strains = x.shape
        S = np.empty((4, B * n_dcc))
        harness.harness_dc_summaries(_ptr(_masks(x).reshape(-1)), ctypes.c_int64(B * n_dcc), n_obs,
                                     n_strains, _ptr(S))
        want = _summ(x)
        for j in (1, 2, 3):
            assert np.array_equal(S[j], want[j].ravel()), j
        # Shannon: the host's log against NumPy's
        np.testing.assert_allclose(S[0], want[0].ravel(), rtol=4e-16, atol=0)
    gd = load_golden('daycare_distance')
    cases = [(gd['sim_small'], list(gd['obs_small'])), (gd['sim_nan'], list(gd['obs_small']))]
    cases.append((gd['sim_small'], [np.zeros((1, 5))] + list(gd['obs_small'][1:])))
    for j in range(20):
        n_ss, n_dcc, B = rs.randint(1, 5), rs.randint(1, 33), rs.randint(1, 4)
        sim = rs.exponential(size=(n_ss, B, n_dcc)) * 10.0 ** rs.uniform(-3, 3, (n_ss, 1, 1))
        obs = list(rs.exponential(size=(n_ss, 1, n_dcc)))
        cases.append((sim, obs))
    from elfi_b200 import ops
    for sim, obs in cases:
        for rows in (slice(None), slice(0, 1)):
            s = np.asarray(sim)[:, rows]
            B, n_dcc = s.shape[1], s.shape[2]
            om, y = ops.daycare_observed(obs)
            d = np.empty(B)
            S = np.ascontiguousarray(s.transpose(1, 0, 2))
            harness.harness_dc_distance(_ptr(S), ctypes.c_int64(B), len(obs), n_dcc, _ptr(om),
                                        _ptr(np.ascontiguousarray(y)), _ptr(d))
            assert np.array_equal(d, dc.distance(*s, observed=obs), equal_nan=True)


def test_replay_matches_header(harness):
    """The NumPy replay of the kernel against the header run on the host from the same draws:
    every DCC's final state, after the replay's K transitions."""
    import streams
    import daycare_replay as rp
    P = np.array([[3.6, 0.6, 0.1], [11.0, 2.0, 1.0], [0.0, 0.6, 0.1], [3.6, 0.6, 0.0]])
    f = SMALL['freq_strains_commun']
    n_dcc, n_ind, n_strains = 5, 12, 6
    masks, K, k_c, _ = rp.simulate(P, n_dcc, n_ind, n_strains, f, 9, 2.0, seed=11, offset=2 ** 32 - 2)
    assert np.array_equal(K, k_c.max(axis=1)) and (K > 0).all()
    rows = streams.rows_of(len(P), 2 ** 32 - 2)
    for b in range(len(P)):
        for c in range(n_dcc):
            ks = np.arange(K[b])
            w = streams.philox4x32_10(rows[b] & np.uint64(0xFFFFFFFF), rows[b] >> np.uint64(32), ks,
                                      rp.SALT_DAYCARE + c, 11)
            E = -np.log(streams.u01(w[0], w[1]))
            x = 1.0 - streams.u01(w[2], w[3])
            m = np.zeros(n_ind, dtype=np.uint64)
            dt = np.empty(K[b])
            num = np.empty(n_strains, dtype=np.int64)
            harness.harness_dc_run(_ptr(m), n_ind, n_strains, _ptr(P[b]), _ptr(f), _ptr(E), _ptr(x),
                                   ctypes.c_int64(K[b]), _ptr(dt), _ptr(num))
            assert np.array_equal(m, masks[b, c]), (b, c)
            t = np.cumsum(dt)
            assert int(np.argmax(t >= 2.0)) + 1 == k_c[b, c]


# ---------------------------------------------------------------------------- Python layer
@pytest.fixture
def dc_double(cpu_double, monkeypatch):
    import abi_double
    import daycare_double
    import priors_double
    abi_double.install(monkeypatch, priors_double.TABLE, daycare_double.TABLE)
    return cpu_double


def test_ops_validate_before_the_call(dc_double):
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    P = np.tile([3.6, 0.6, 0.1], (3, 1))
    for kw, msg in ((dict(n_dcc=33), 'n_dcc'), (dict(n_dcc=0), 'n_dcc'), (dict(n_ind=65), 'n_ind'),
                    (dict(n_ind=1, n_obs=1), 'n_ind'), (dict(n_strains=41), 'n_strains'),
                    (dict(n_obs=54), 'n_obs'), (dict(n_obs=0), 'n_obs'),
                    (dict(time_end=0.0), 'time_end'), (dict(time_end=np.inf), 'time_end'),
                    (dict(time_end=np.nan), 'time_end'),
                    (dict(freq_strains_commun=np.full(32, 0.1)), 'freq_strains_commun'),
                    (dict(n_strains=2, freq_strains_commun=[0.1, -0.1]), 'finite and >= 0'),
                    (dict(n_strains=2, freq_strains_commun=[0.1, np.nan]), 'finite and >= 0'),
                    (dict(n_strains=2, freq_strains_commun=[np.inf, 0.1]), 'finite and >= 0')):
        with pytest.raises(ValueError, match=msg):
            ops.sim_daycare(P, **kw)
    with pytest.raises(ValueError, match='parameter width of 2'):
        ops.sim_daycare(P[:, :2])
    with pytest.raises(ValueError, match='n_strains'):
        ops.daycare_summaries(dev.to_device(np.zeros((2, 3, 4, 65))))
    with pytest.raises(ValueError, match='batch, n_dcc, n_obs, n_strains'):
        ops.daycare_summaries(dev.to_device(np.zeros((2, 3, 4))))
    with pytest.raises(ValueError, match='at most 128'):
        ops.daycare_distance(dev.to_device(np.zeros((2, 5 * 29))), [np.zeros((1, 29))] * 5, 29)
    assert not dc_double.CALLS


def test_dispatch_host_device_and_lazy_agree(dc_double):
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    from elfi_b200.examples import daycare as dc
    g = load_golden('daycare_draws')
    x = g['mixed']
    fns = (dc.ss_shannon, dc.ss_strains, dc.ss_prevalence, dc.ss_prevalence_multi)
    h = _summ(x)
    xd = dev.to_device(x.astype(np.float64)) != 0
    for j, fn in enumerate(fns):
        assert np.array_equal(fn(xd).cpu().numpy(), h[j]), j
    assert np.array_equal(ops.daycare_summaries(x).cpu().numpy(), np.concatenate(h, axis=1))
    obs = _summ(g['small1'])
    dd = dc.distance(*[fn(xd) for fn in fns], observed=obs)
    assert np.array_equal(dd.cpu().numpy(), dc.distance(*h, observed=obs))
    lazy = dc.daycare_device(np.array([3.6, -1.0, 11.0]), 0.6, 0.1, batch_size=3,
                             random_state=np.random.RandomState(1), **SMALL)
    assert lazy.shape == (3, 5, 9, 6)
    data = lazy.materialize().cpu().numpy()
    S = [fn(lazy).cpu().numpy() for fn in fns]
    want = _summ(data)
    for j in range(4):
        assert np.isnan(S[j][1]).all()
        assert np.array_equal(S[j][[0, 2]], want[j][[0, 2]]), j
    assert dc_double.CALLS.count('elfi_b200_sim_daycare_f64') == 2
    S, X, K = ops.sim_daycare(np.array([[3.6, 0.6, 0.1], [np.nan, 0.6, 0.1], [np.inf, 0.6, 0.1],
                                        [3.6, 1e300, 0.1]]), want_data=True, **SMALL)
    K = K.cpu().numpy()
    assert K[0] > 0 and (K[1:] == -1).all() and not X.cpu().numpy()[1:].any()
    assert np.isnan(S.cpu().numpy()[1:]).all()


def test_device_model_runs_rejection_smc_and_bolfi(dc_double):
    import elfi_b200 as elfi
    from elfi_b200.examples import daycare as dc
    m, dp = dc.get_device_model(seed_obs=3, **SMALL)
    host_m = dc.get_model(seed_obs=3, **SMALL)
    assert np.array_equal(m.observed['DCC'], host_m.observed['DCC'])
    assert sorted(n for n in m.nodes if not n.startswith('_')) == sorted(
        n for n in host_m.nodes if not n.startswith('_'))
    res = elfi.Rejection(m['d'], batch_size=20, seed=1).sample(5, quantile=0.25, bar=False)
    assert res.n_samples == 5 and not np.any(np.isnan(res.discrepancies))
    smc = elfi.SMC(m['d'], batch_size=20, seed=2, device_proposal=dp).sample(
        5, quantiles=[0.5, 0.5], bar=False)
    assert len(smc.populations) == 2
    assert 'elfi_b200_sim_daycare_f64' in dc_double.CALLS
    assert 'elfi_b200_daycare_distance_f64' in dc_double.CALLS
