"""GPU checks of the n-D Gaussian mean model (elfi_b200/csrc/gauss_nd.cu).

* the summary kernel bit for bit against np.mean / np.var(axis=1) at D in {1, 2, 3, 7, 8, 9, 16,
  33} and n in {1, 2, 15, 50, 1000}, on contiguous, strided and transposed views, NaN and inf;
* the distance bit for bit against the reference's euclidean_multidim up to D = 300;
* the host model on the device against the reference's goldens: generate and Rejection bit for bit,
  SMC at the SMC parity bar;
* the device simulator: every element within the replay's bound (tests/gauss_nd_replay.py), fused
  summaries equal to the summary kernel of the written data bit for bit, rows that do not depend on
  the launch, the law of the summaries against the host simulator, and SMC near the true means;
* the reference's test_gauss_1d_mean and test_gauss_2d_mean in both modes.
"""
import numpy as np
import pytest
import scipy.stats as ss

import gauss_nd_replay as gr
from conftest import load_golden
from mahalanobis_cases import ATOL, RTOL, same_bits
from test_gauss_nd_host import (CONFIGS, DIMS, DIST_DIMS, NOBS, REJECTION, SEED_OBS,
                                SMC_THRESHOLDS, THRESHOLD, crafted)

pytestmark = [pytest.mark.gpu, pytest.mark.first_device_run]


def _host(x):
    from elfi_b200 import device as dev
    return np.asarray(dev.to_host(x))


def _np_meanvar(y):
    y = np.ascontiguousarray(y)
    with np.errstate(invalid='ignore'):
        return np.mean(y, axis=1), np.var(y, axis=1)


# ---------------------------------------------------------------------------- summaries, distance
@pytest.mark.parametrize('D', DIMS)
def test_summaries_bit_for_bit_numpy(D):
    import torch
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    rs = np.random.RandomState(100 + D)
    for n in NOBS:
        y = crafted(37, n, D, rs)
        mean, var = _np_meanvar(y)
        views = {'contiguous': dev.to_device(y)}
        big = dev.to_device(np.concatenate([y, y[:, :, :1]], axis=2).repeat(2, axis=1))
        views['strided'] = big[:, ::2, :D]
        views['transposed'] = dev.to_device(np.ascontiguousarray(y.transpose(2, 1, 0))).permute(2, 1, 0)
        views['host'] = y
        for name, v in views.items():
            if isinstance(v, torch.Tensor):
                assert np.array_equal(_host(v), y, equal_nan=True), name
            S = _host(ops.gauss_nd_summaries(v))
            assert same_bits(S[:, :D], mean), (n, name)
            assert same_bits(S[:, D:], var), (n, name)


@pytest.mark.parametrize('D', DIST_DIMS)
def test_distance_bit_for_bit_reference(D):
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    from elfi_b200.examples import gauss
    rs = np.random.RandomState(D)
    S = rs.randn(5003, D) * np.exp(rs.randn(5003, D) * 3)
    obs = rs.randn(1, D)
    S[0, 0], S[1, D - 1], S[2, 0], S[3] = np.nan, np.inf, -np.inf, obs[0]
    with np.errstate(invalid='ignore'):
        want = gauss.euclidean_multidim(S, observed=[obs])
    assert same_bits(_host(ops.gauss_nd_distance(S, obs)), want)
    wide = dev.to_device(np.concatenate([S, S], axis=1))
    assert same_bits(_host(gauss.euclidean_multidim(wide[:, :D], observed=[dev.to_device(obs)])),
                     want)
    T = dev.to_device(np.ascontiguousarray(S.T)).t()
    assert same_bits(_host(ops.gauss_nd_distance(T, obs)), want)


# ---------------------------------------------------------------------------- host model goldens
def _model(tag):
    from elfi_b200.examples import gauss
    tp, cov = CONFIGS[tag]
    return gauss.get_model(true_params=tp, seed_obs=SEED_OBS[tag], nd_mean=True, cov_matrix=cov)


@pytest.mark.parametrize('tag', sorted(CONFIGS))
def test_host_model_matches_reference_golden(tag):
    import elfi_b200 as elfi
    g = load_golden('gauss_nd')
    names = ['mu_{}'.format(i) for i in range(len(CONFIGS[tag][0]))]
    m = _model(tag)
    assert same_bits(m.observed['gauss'], g[tag + '_observed'])
    out = m.generate(20, seed=11)
    for k in names + ['gauss', 'ss_mean', 'ss_var', 'd']:
        assert same_bits(_host(out[k]), g['{}_gen_{}'.format(tag, k)]), k
    for run, (init, kw) in sorted(REJECTION.items()):
        if run == 'threshold':
            kw = dict(kw, threshold=THRESHOLD[tag])
        res = elfi.Rejection(m['d'], **init).sample(bar=False, **kw)
        pre = '{}_{}_'.format(tag, run)
        assert res.n_sim == int(g[pre + 'n_sim']), run
        assert res.threshold == float(g[pre + 'threshold']), run
        assert same_bits(res.discrepancies, g[pre + 'd']), run
        for k in names:
            assert same_bits(res.samples[k], g[pre + k]), (run, k)
    res = elfi.SMC(m['d'], batch_size=1000, seed=20).sample(150, thresholds=SMC_THRESHOLDS[tag],
                                                           bar=False)
    pre = tag + '_smc_'
    assert res.n_sim == int(g[pre + 'n_sim'])
    for i, pop in enumerate(res.populations):
        p = '{}pop{}_'.format(pre, i)
        for k, v in dict({k: pop.samples[k] for k in names}, d=pop.discrepancies).items():
            if i == 0:
                assert same_bits(v, g[p + k]), (i, k)
            else:
                np.testing.assert_allclose(v, g[p + k], rtol=RTOL, atol=ATOL, err_msg=str((i, k)))
    np.testing.assert_allclose(res.discrepancies, g[pre + 'd'], rtol=RTOL, atol=ATOL)


# ---------------------------------------------------------------------------- device simulator
@pytest.mark.parametrize('D', (1, 2, 3, 7, 16))
@pytest.mark.parametrize('offset', (0, 2 ** 32 - 300))
def test_sim_matches_replay(D, offset):
    from elfi_b200 import ops
    rs = np.random.RandomState(D)
    C = rs.randn(D, D)
    A = ops.gauss_nd_factor(C @ C.T / D + np.eye(D), D)
    mu = rs.uniform(-5, 5, (700, D))
    for n_obs in (1, 15, 50):
        Y = _host(ops.sim_gauss_nd(mu, A, n_obs, seed=77, offset=offset, want_data=True,
                                   want_summaries=False)[0])
        want, err = gr.sim_gauss_nd(mu, A, n_obs, seed=77, offset=offset)
        assert Y.shape == (700, n_obs, D)
        bad = np.abs(Y - want) > err
        assert not bad.any(), (n_obs, np.argwhere(bad)[:3], np.max(np.abs(Y - want)))


@pytest.mark.parametrize('D', (1, 2, 16))
def test_fused_summaries_equal_summary_kernel(D):
    from elfi_b200 import device as dev
    from elfi_b200 import ops
    rs = np.random.RandomState(D)
    A = ops.gauss_nd_factor(np.eye(D) + 0.3, D)
    B = 100003
    mu = dev.to_device(rs.uniform(-5, 5, (B, 2 * D)))[:, ::2]       # strided means
    for n_obs in (1, 15, 50, 129):
        Y, S = ops.sim_gauss_nd(mu, A, n_obs, seed=5, want_data=True)
        _, S2 = ops.sim_gauss_nd(mu, A, n_obs, seed=5)
        assert same_bits(_host(S), _host(ops.gauss_nd_summaries(Y))), n_obs
        assert same_bits(_host(S2), _host(S)), n_obs


def test_rows_do_not_depend_on_the_launch():
    from elfi_b200 import ops
    rs = np.random.RandomState(3)
    for D in (1, 3, 16):
        A = ops.gauss_nd_factor(None, D)
        mu = rs.uniform(-5, 5, (1000, D))
        Y, S = ops.sim_gauss_nd(mu, A, 17, seed=9, offset=2 ** 32 - 500, want_data=True)
        cols = [mu[700:, j] for j in range(D)]
        Y2, S2 = ops.sim_gauss_nd(cols, A, 17, seed=9, offset=2 ** 32 + 200, want_data=True)
        assert same_bits(_host(Y)[700:], _host(Y2)), D
        assert same_bits(_host(S)[700:], _host(S2)), D


@pytest.mark.parametrize('D,cov', [(1, [1]), (2, [[1, .5], [.5, 1]]), (3, [[1, 1, 0], [1, 1, 0],
                                                                           [0, 0, 2]])])
def test_law_of_the_summaries_matches_host(D, cov):
    """ss_mean and ss_var of the device simulator against the reference's SciPy simulator, per
    coordinate (a singular covariance included)."""
    from elfi_b200 import ops
    from elfi_b200.examples import gauss
    mu = np.arange(1.0, D + 1)
    n_obs = 15
    host = gauss.gauss_nd_mean(*mu, cov_matrix=cov, n_obs=n_obs, batch_size=3000,
                               random_state=np.random.RandomState(1))
    hm, hv = np.mean(host, axis=1), np.var(host, axis=1)
    S = _host(ops.sim_gauss_nd(np.tile(mu, (30000, 1)), ops.gauss_nd_factor(cov, D), n_obs,
                               seed=2)[1])
    for j in range(D):
        assert ss.ks_2samp(S[:, j], hm[:, j]).pvalue > 1e-3, ('mean', j)
        assert ss.ks_2samp(S[:, D + j], hv[:, j]).pvalue > 1e-3, ('var', j)
    if D == 3:
        A = ops.gauss_nd_factor(cov, D)
        Y = _host(ops.sim_gauss_nd(np.tile(mu, (2000, 1)), A, 50, seed=3, want_data=True,
                                   want_summaries=False)[0])
        # cov [[1, 1], [1, 1]] in the first two coordinates: equal deviations from the means, up to
        # the square root of the rounding-level singular value in NumPy's factor (about 1e-8)
        gap = np.abs(A[:, 0] - A[:, 1]).sum()
        assert gap < 1e-6
        assert np.all(np.abs((Y[:, :, 0] - mu[0]) - (Y[:, :, 1] - mu[1])) <= 10 * gap + 1e-12)


def test_device_model_smc_near_the_true_means():
    import elfi_b200 as elfi
    from elfi_b200.examples import gauss
    rs = np.random.RandomState(0)
    true = list(rs.uniform(-3, 3, 16))
    C = rs.randn(16, 16) * 0.2
    cov = C @ C.T + np.eye(16)
    m, dp = gauss.get_device_model(true_params=true, seed_obs=4, nd_mean=True, cov_matrix=cov)
    res = elfi.SMC(m['d'], batch_size=100000, seed=6, device_proposal=dp).sample(
        2000, thresholds=[8.0, 5.0, 3.5, 2.5, 2.0], bar=False)
    assert len(res.populations) == 5 and np.all(np.isfinite(res.weights))
    post = np.array([np.average(res.samples['mu_{}'.format(i)], weights=res.weights)
                     for i in range(16)])
    obs_mean = np.mean(m.observed['gauss'][0], axis=0)
    assert np.all(np.abs(post - obs_mean) < 0.6), post - obs_mean
    assert res.discrepancies.max() <= 2.0


def test_reference_gauss_1d_and_2d_mean_both_modes():
    """The reference's test_gauss_1d_mean and test_gauss_2d_mean, with the host model and with the
    device model."""
    import elfi_b200 as elfi
    from elfi_b200.examples import gauss
    for params_true, cov_matrix in (([4], [1]), ([4, 4], [[1, .5], [.5, 1]])):
        m = gauss.get_model(true_params=params_true, nd_mean=True, cov_matrix=cov_matrix)
        res = elfi.Rejection(m, m['d'], batch_size=10).sample(20, bar=False)
        assert len(res.samples['mu_0']) == 20
        md, dp = gauss.get_device_model(true_params=params_true, nd_mean=True,
                                        cov_matrix=cov_matrix)
        res = elfi.Rejection(md, md['d'], batch_size=10).sample(20, bar=False)
        assert len(res.samples['mu_0']) == 20
        assert np.all(np.abs(np.asarray(res.samples['mu_0']) - 4) <= 5)
