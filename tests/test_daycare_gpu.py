"""Device day care simulator, summaries and distance.

* per-row replay (tests/daycare_replay.py over oracle/streams.py): K and the observed states equal
  the kernel's exactly, except for rows where the replay finds a DCC's time within MARGIN (relative)
  of time_end (the device's log against NumPy's); at the default size for the truth, prior draws and
  the box corners, and at a reduced size for invalid rows, row counters across 2^32 and a batch that
  is not a multiple of the CTA count; every row's K is the largest of its DCCs' crossing counts;
* split launches equal one launch; the fused summaries equal daycare_summaries of the written data
  bit for bit, and NumPy's but for Shannon's log (within SHANNON_ULPS), on strided views too;
* daycare_distance equals the reference's distance bit for bit for B = 1 and B > 1;
* statistics against the host simulator at batch_size=1, Rejection posteriors against the host
  model, SMC determinism and a short BOLFI run on logd.
"""
import numpy as np
import pytest
import scipy.stats as ss

import daycare_replay as rp
from conftest import load_golden

pytestmark = pytest.mark.gpu
TRUTH = [3.6, 0.6, 0.1]
DEFAULT = dict(n_dcc=29, n_ind=53, n_strains=33, n_obs=36, time_end=10.)
SMALL = dict(n_dcc=5, n_ind=12, n_strains=6, n_obs=9, time_end=2.0,
             freq_strains_commun=np.array([0.05, 0.1, 0.2, 0.02, 0.3, 0.15]))
REDUCED = dict(n_dcc=10, n_ind=20, n_strains=8, n_obs=15, time_end=2.0)
MARGIN = 1e-12
SHANNON_ULPS = 2   # the device's log and NumPy's are each within 1 ulp


def _np(t):
    return t.cpu().numpy()


def _summ(x):
    from elfi_b200.examples import daycare as dc
    return np.concatenate([dc.ss_shannon(x), dc.ss_strains(x), dc.ss_prevalence(x),
                           dc.ss_prevalence_multi(x)], axis=1)


def _prior(B, seed):
    rs = np.random.RandomState(seed)
    return np.column_stack([rs.uniform(0, 11, B), rs.uniform(0, 2, B), rs.uniform(0, 1, B)])


def _check_replay(P, cfg, seed, offset=0):
    from elfi_b200 import ops
    f = cfg.get('freq_strains_commun')
    f = np.full(cfg['n_strains'], 0.1) if f is None else f
    S, X, K = ops.sim_daycare(P, seed=seed, offset=offset, want_data=True, **cfg)
    masks, K_r, k_c, margin = rp.simulate(P, cfg['n_dcc'], cfg['n_ind'], cfg['n_strains'], f,
                                          cfg['n_obs'], cfg['time_end'], seed, offset)
    data_r = rp.data_of(masks, cfg['n_obs'], cfg['n_strains'])
    K, X = _np(K), _np(X)
    excused = margin < MARGIN
    print('replay: {} rows, {} excused (a time within {} of time_end), smallest margin {:.3g}'
          .format(len(P), int(excused.sum()), MARGIN, margin.min()))
    ok = ~excused
    assert np.array_equal(K[ok], K_r[ok])
    assert np.array_equal(X[ok], data_r[ok])
    valid = K_r >= 0
    assert np.array_equal(K_r[valid], k_c[valid].max(axis=1))
    assert (k_c[valid] >= 1).all()
    return S, X, K


def test_replay_default_size_truth_prior_and_corners():
    P = np.vstack([np.tile(TRUTH, (3, 1)), _prior(6, 1),
                   [[0.0, 0.6, 0.1], [3.6, 0.0, 0.1], [3.6, 0.6, 0.0], [0.0, 0.0, 0.0],
                    [11.0, 2.0, 1.0]]])
    _check_replay(P, DEFAULT, seed=5)


@pytest.mark.parametrize('offset', [0, 2 ** 32 - 20])
def test_replay_small_invalid_rows_and_odd_batch(offset):
    P = np.vstack([_prior(33, 2), [[-1.0, 0.6, 0.1], [3.6, np.nan, 0.1], [3.6, 0.6, -0.5],
                                   [np.inf, 0.6, 0.1], [3.6, np.inf, 0.1], [3.6, 0.6, np.inf],
                                   [1e300, 0.6, 0.1], [3.6, 0.6, 1e300]],
                   [[11.0, 2.0, 1.0]]])
    S, X, K = _check_replay(P, SMALL, seed=7, offset=offset)
    assert (K[33:41] == -1).all() and np.isnan(_np(S)[33:41]).all() and not X[33:41].any()
    assert (K[[*range(33), 41]] > 0).all()


@pytest.mark.parametrize('B', [1, 257])
def test_split_launches_equal_one_launch(B):
    from elfi_b200 import ops
    P = _prior(B, 3)
    S, X, K = ops.sim_daycare(P, seed=9, offset=100, want_data=True, **REDUCED)
    k = B // 3
    S1, X1, K1 = ops.sim_daycare(P[:k], seed=9, offset=100, want_data=True, **REDUCED)
    S2, X2, K2 = ops.sim_daycare(P[k:], seed=9, offset=100 + k, want_data=True, **REDUCED)
    assert np.array_equal(_np(S), np.concatenate([_np(S1), _np(S2)]), equal_nan=True)
    assert np.array_equal(_np(X), np.concatenate([_np(X1), _np(X2)]))
    assert np.array_equal(_np(K), np.concatenate([_np(K1), _np(K2)]))


def _ulps(a, b):
    return np.abs(a - b) / np.spacing(np.maximum(np.abs(a), np.abs(b)))


@pytest.mark.parametrize('cfg', [DEFAULT, SMALL, REDUCED])
def test_fused_equals_unfused_and_numpy(cfg):
    import torch
    from elfi_b200 import ops
    P = np.vstack([_prior(3000, 4), [[0.0, 0.0, 0.0]]])
    S, X, _ = ops.sim_daycare(P, seed=2, want_data=True, **cfg)
    S_only = ops.sim_daycare(P, seed=2, **cfg)[0]
    assert np.array_equal(_np(S), _np(S_only))
    assert np.array_equal(_np(ops.daycare_summaries(X)), _np(S))
    B, n_dcc, n_obs, n_strains = X.shape
    big = torch.zeros((B, n_dcc + 1, n_obs + 2, n_strains + 3), dtype=torch.uint8, device='cuda')
    view = big[:, 1:, 2:, 3:]
    view.copy_(X)
    assert np.array_equal(_np(ops.daycare_summaries(view)), _np(S))
    got, want = _np(S), _summ(_np(X))
    assert np.array_equal(got[:, n_dcc:], want[:, n_dcc:])
    sh_g, sh_w = got[:, :n_dcc], want[:, :n_dcc]
    diff = sh_g != sh_w
    print('Shannon: {} of {} differ from NumPy, at most {} ulps'.format(
        int(diff.sum()), diff.size, _ulps(sh_g[diff], sh_w[diff]).max() if diff.any() else 0))
    assert (_ulps(sh_g[diff], sh_w[diff]) <= SHANNON_ULPS).all()


def test_summaries_of_crafted_data_equal_reference():
    from elfi_b200 import ops
    g = load_golden('daycare_summaries')
    for name in ('zeros', 'diag', 'ones'):
        got = _np(ops.daycare_summaries(g['x_' + name]))
        n_dcc = g['x_' + name].shape[1]
        for j in range(4):
            assert np.array_equal(got[:, j * n_dcc:(j + 1) * n_dcc], g[name][j]), (name, j)


def test_distance_equals_reference():
    from elfi_b200 import device as dev
    from elfi_b200.examples import daycare as dc
    gd = load_golden('daycare_distance')
    gs = load_golden('daycare_summaries')
    obs = list(gs['truth1'][:, :, :])
    obs = [o.reshape(1, -1) for o in obs]
    sim = [dev.to_device(s) for s in gs['truth2']]
    assert np.array_equal(_np(dc.distance(*sim, observed=obs)), gd['d_truth_b2'])
    assert np.array_equal(_np(dc.distance(*[s[:1] for s in sim], observed=obs)), gd['d_truth_b1'])
    assert np.array_equal(_np(dc.distance(*[s[1:] for s in sim], observed=obs)),
                          gd['d_truth_b1_row1'])
    obs_s = list(gd['obs_small'])
    for key, o in (('d_small', obs_s), ('d_small_obs0', [np.zeros((1, 5))] + obs_s[1:])):
        got = dc.distance(*[dev.to_device(s) for s in gd['sim_small']], observed=o)
        assert np.array_equal(_np(got), gd[key]), key
    got = dc.distance(*[dev.to_device(s) for s in gd['sim_nan']], observed=obs_s)
    assert np.array_equal(_np(got), gd['d_nan'], equal_nan=True)
    rs = np.random.RandomState(5)
    for n_dcc in (1, 7, 29, 32):
        o = [rs.exponential(size=(1, n_dcc)) for _ in range(4)]
        for B in (1, 2, 1001):
            s = [rs.exponential(size=(B, n_dcc)) * 10.0 ** rs.uniform(-2, 2) for _ in range(4)]
            got = dc.distance(*[dev.to_device(v) for v in s], observed=o)
            assert np.array_equal(_np(got), dc.distance(*s, observed=o)), (n_dcc, B)


def test_statistics_match_host_simulator():
    """KS tests of each summary's DCC mean: device rows against the host simulator at
    batch_size=1."""
    from elfi_b200 import ops
    from elfi_b200.examples import daycare as dc
    n = 300
    rs = np.random.RandomState(6)
    for prm in (TRUTH, [8.0, 1.0, 0.5]):
        host = np.concatenate([_summ(dc.daycare(*prm, random_state=rs, **REDUCED))
                               for _ in range(n)])
        S = _np(ops.sim_daycare(np.tile(prm, (20000, 1)), seed=11, **REDUCED)[0])
        k = REDUCED['n_dcc']
        for j in range(4):
            p = ss.ks_2samp(S[:, j * k:(j + 1) * k].mean(axis=1),
                            host[:, j * k:(j + 1) * k].mean(axis=1)).pvalue
            assert p > 1e-4, (prm, j, p)


def test_device_rejection_posterior_matches_host():
    import elfi_b200 as elfi
    from elfi_b200.examples import daycare as dc
    host_m = dc.get_model(seed_obs=2, **SMALL)
    res_h = elfi.Rejection(host_m['d'], batch_size=1, seed=1).sample(60, quantile=0.05, bar=False)
    m, dp = dc.get_device_model(seed_obs=2, **SMALL)
    assert np.array_equal(m.observed['DCC'], host_m.observed['DCC'])
    res_d = elfi.Rejection(m['d'], batch_size=100000, seed=1).sample(5000, quantile=0.05,
                                                                     bar=False)
    for name in ('t1', 't2', 't3'):
        h, d = res_h.samples[name], res_d.samples[name]
        se = np.sqrt(h.var() / len(h) + d.var() / len(d))
        assert abs(h.mean() - d.mean()) < 4.5 * se, (name, h.mean(), d.mean(), se)


def test_device_model_smc_and_bolfi():
    import elfi_b200 as elfi
    from elfi_b200.examples import daycare as dc
    m, dp = dc.get_device_model(seed_obs=3, time_end=2.0)

    def run(**kw):
        return elfi.SMC(m['d'], batch_size=5000, seed=4, device_proposal=dp, **kw).sample(
            200, quantiles=[0.1, 0.3], bar=False)
    smc = run()
    assert len(smc.populations) == 2 and np.all(np.isfinite(smc.weights))
    par = run(distributed=False, max_parallel_batches=2)
    par2 = run(distributed=False, max_parallel_batches=2)
    assert np.array_equal(par.samples_array, par2.samples_array)
    assert np.array_equal(par.weights, par2.weights)
    bolfi = elfi.BOLFI(m['logd'], batch_size=5, initial_evidence=20, update_interval=10,
                       bounds={'t1': (0, 11), 't2': (0, 2), 't3': (0, 1)}, seed=1)
    bolfi.fit(n_evidence=40, bar=False)
    assert bolfi.n_evidence == 40
