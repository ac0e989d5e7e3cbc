"""Device scratch assay simulator.

* sim_scratch_assay equals the NumPy replay of its Philox streams (tests/scratch_assay_replay.py)
  bit for bit, frames and summaries, at the default and reduced sizes and at row counters across
  2^32; split launches equal one launch;
* the fused summaries equal scratch_assay_summaries of the written frames (strided views too) and
  NumPy's cell_summaries of the materialised data; full and empty lattices;
* the Rejection posterior of the device model against the host model's, and the samplers.
"""
import numpy as np
import pytest

import scratch_assay_replay as rp
from conftest import load_golden

pytestmark = pytest.mark.gpu
REDUCED = [8, 10, 20, 3]
EDGES = [[0.25, 0.002], [0.0, 0.0], [0.0, 1.0], [1.0, 0.0], [1.0, 1.0], [1.5, -0.5],
         [np.nan, 0.3], [0.3, np.nan], [0.9, 0.5]]


def _np(t):
    return t.cpu().numpy()


def _default_init():
    return load_golden('scratch_assay_draws')['obs'][0, :, :, 0]


def _reduced_init():
    from elfi_b200.examples import scratch_assay as sa
    return sa._random_init(*REDUCED, random_state=np.random.RandomState(1))


@pytest.mark.parametrize('offset', [0, 2 ** 32 - 5])
def test_sim_equals_replay_at_the_default_size(offset):
    from elfi_b200 import ops
    init = _default_init()
    P = np.array(EDGES[:5] + [[0.05, 0.01], [0.4, 0.02]])
    X, S = ops.sim_scratch_assay(P, init, seed=13, offset=offset, want_data=True)
    Xr, Sr = rp.sim(P, init, 144, 2, seed=13, offset=offset)
    assert np.array_equal(_np(X), Xr.astype(bool))
    assert np.array_equal(_np(S), Sr)


@pytest.mark.parametrize('offset', [0, 2 ** 32 - 40])
def test_sim_equals_replay_at_the_reduced_size(offset):
    from elfi_b200 import ops
    init = _reduced_init()
    rs = np.random.RandomState(offset % 97)
    P = np.vstack([EDGES, rs.uniform(0, 1, (71, 2))])
    X, S = ops.sim_scratch_assay(P, init, seed=3, offset=offset, want_data=True)
    Xr, Sr = rp.sim(P, init, 144, 2, seed=3, offset=offset)
    assert np.array_equal(_np(X), Xr.astype(bool))
    assert np.array_equal(_np(S), Sr)
    # other observation spacings
    X, S = ops.sim_scratch_assay(P[:12], init, obs_period=2, obs_interval=1 / 8, tau=1 / 24,
                                 seed=3, offset=offset, want_data=True)
    Xr, Sr = rp.sim(P[:12], init, 16, 3, seed=3, offset=offset)
    assert np.array_equal(_np(X), Xr.astype(bool)) and np.array_equal(_np(S), Sr)


def test_split_launches_equal_one_launch():
    from elfi_b200 import ops
    init = _reduced_init()
    P = np.random.RandomState(2).uniform(0, 1, (1000, 2))
    base = 2 ** 32 - 300
    whole = ops.sim_scratch_assay(P, init, seed=9, offset=base, want_data=True)
    for cut in (1, 300, 777):
        parts = [ops.sim_scratch_assay(P[:cut], init, seed=9, offset=base, want_data=True),
                 ops.sim_scratch_assay(P[cut:], init, seed=9, offset=base + cut, want_data=True)]
        for j in range(2):
            joined = np.concatenate([_np(parts[0][j]), _np(parts[1][j])])
            assert np.array_equal(joined, _np(whole[j])), (cut, j)


@pytest.mark.parametrize('B', [1, 129, 20011])
def test_fused_summaries_equal_unfused_chain(B):
    from elfi_b200 import ops
    from elfi_b200.examples import scratch_assay as sa
    init = _default_init()
    rs = np.random.RandomState(B)
    P = rs.uniform(0, 1, (B, 2))
    P[::3, 1] *= 0.02
    X, S = ops.sim_scratch_assay(P, init, seed=5, offset=2 ** 32 - 50, want_data=True)
    _, S_only = ops.sim_scratch_assay(P, init, seed=5, offset=2 ** 32 - 50)
    S = _np(S)
    assert np.array_equal(_np(S_only), S)
    assert np.array_equal(_np(ops.scratch_assay_summaries(X)), S)
    if B <= 129:
        x = _np(X)
        assert np.array_equal(sa.cell_summaries(x.astype(np.float64)), S)
        assert np.array_equal(_np(sa.cell_summaries(X)), S)
        # a strided view: every other frame of a column-major copy
        Xt = X.permute(3, 1, 2, 0).contiguous().permute(3, 1, 2, 0)[..., ::2]
        assert np.array_equal(_np(ops.scratch_assay_summaries(Xt)),
                              sa.cell_summaries(x[..., ::2].astype(np.float64)))


def test_summaries_of_golden_arrays():
    from elfi_b200 import ops
    g = load_golden('scratch_assay_summaries')
    d = load_golden('scratch_assay_draws')
    for name, arr in (('obs', d['obs']), ('batch', d['batch']), ('fill', d['fill'][None]),
                      ('empty', d['empty'][None]), ('reduced', d['reduced'][None]),
                      ('crafted', g['crafted'])):
        assert np.array_equal(_np(ops.scratch_assay_summaries(arr)), g[name + '_sums']), name


def test_full_and_empty_lattices():
    from elfi_b200 import ops
    P = np.array([[0.5, 0.5], [1.0, 1.0], [0.0, 0.0]])
    for init, count in ((np.ones((27, 36)), 972), (np.zeros((27, 36)), 0),
                        (np.ones((64, 64)), 4096)):
        X, S = ops.sim_scratch_assay(P, init, seed=1, want_data=True)
        X, S = _np(X), _np(S)
        assert np.all(X == (init[None, :, :, None] != 0)) and np.all(S[:, :-1] == 0)
        assert np.all(S[:, -1] == count)
    # a lattice that fills: the rows finish early with the frames the replay has
    init = _default_init()
    P = np.array([[0.3, 1.0], [0.0, 0.9]])
    X, S = ops.sim_scratch_assay(P, init, seed=4, want_data=True)
    Xr, Sr = rp.sim(P, init, 144, 2, seed=4)
    assert np.array_equal(_np(X), Xr.astype(bool)) and np.array_equal(_np(S), Sr)
    assert np.all(Sr[:, -1] == 972)


def test_device_rejection_posterior_matches_host():
    import elfi_b200 as elfi
    from elfi_b200.examples import scratch_assay as sa
    host_m = sa.get_model(init_params=REDUCED, seed_obs=2)
    res_h = elfi.Rejection(host_m['d'], batch_size=100, seed=1).sample(40, quantile=0.1,
                                                                       bar=False)
    m, dp = sa.get_device_model(init_params=REDUCED, seed_obs=2)
    assert np.array_equal(m.observed['sim'], host_m.observed['sim'])
    # both keep the best 10 % of whole batches
    res_d = elfi.Rejection(m['d'], batch_size=50000, seed=1).sample(5000, quantile=0.1, bar=False)
    assert res_h.n_sim == 400 and res_d.n_sim == 50000
    for name in ('pm', 'pp'):
        h, d = res_h.samples[name], res_d.samples[name]
        se = np.sqrt(h.var() / len(h) + d.var() / len(d))
        assert abs(h.mean() - d.mean()) < 4 * se, (name, h.mean(), d.mean(), se)


def test_device_model_smc_and_adaptive_distance_smc():
    import elfi_b200 as elfi
    from elfi_b200.examples import scratch_assay as sa
    m, dp = sa.get_device_model(seed_obs=3)
    assert dp.parameter_names == ['pm', 'pp']

    def in_box(s):
        return np.all((s['pm'] >= 0) & (s['pm'] <= 1) & (s['pp'] >= 0) & (s['pp'] <= 1))
    smc = elfi.SMC(m['d'], batch_size=10000, seed=4, device_proposal=dp).sample(
        1000, quantiles=[0.1, 0.3], bar=False)
    assert len(smc.populations) == 2 and np.all(np.isfinite(smc.weights)) and in_box(smc.samples)
    m['d'].become(elfi.AdaptiveDistance(m['sums']))
    ad = elfi.AdaptiveDistanceSMC(m['d'], batch_size=10000, seed=5, device_proposal=dp).sample(
        1000, rounds=2, quantile=0.3, bar=False)
    assert len(ad.populations) == 2 and np.all(np.isfinite(ad.samples_array)) and in_box(ad.samples)
