"""Regression adjustment on the device: ops.linear_adjust against the NumPy restatement
(tests/linadjust_double.py) over shapes, strides and masks; the reference's goldens and functional
tests (tests/golden/gen_golden_post_processing.py); a conjugate Gaussian against its closed form;
and the device MA2 model at about 1e6 accepted rows."""
from functools import partial

import numpy as np
import pytest
import torch

import elfi_b200 as elfi
import linadjust_double as ld
from post_processing_cases import case, check_case, close, statistics
from elfi_b200 import ops, results
from elfi_b200.examples import gauss, ma2
from elfi_b200.post_processing import LinearAdjustment, adjust_posterior

pytestmark = pytest.mark.gpu

QS = (1, 2, 31, 32, 33, 100, 254)
PS = (1, 2, 16)
NS = (2, 3, 255, 256, 257, 10 ** 4, 10 ** 6)


def summaries(N, q, rs, cond=1e3):
    """(N, q) summaries whose centred columns have condition number `cond` when N > q (centred
    orthonormal columns, scaled, rotated and shifted); plain draws otherwise (rank N - 1)."""
    if N <= q:
        return rs.randn(N, q) * 3 + rs.randn(q)
    Q, _ = np.linalg.qr(np.column_stack([np.ones(N), rs.randn(N, q)]))
    rot, _ = np.linalg.qr(rs.randn(q, q))
    return (Q[:, 1:] * np.geomspace(1.0, cond, q) * np.sqrt(N)) @ rot + rs.randn(q)


def thetas(S, p, rs):
    B = rs.randn(S.shape[1], p) / np.sqrt(S.shape[1])
    return (S - S.mean(axis=0)) @ B / S.std() + rs.randn(p) + 0.5 * rs.randn(S.shape[0], p)


def check(S, T, o, adjusted, fits, full_rank=True):
    ref_adj, ref_fits = ld.linear_adjust(S, T, o)
    for k in range(T.shape[1]):
        got = adjusted[k].cpu().numpy()
        close(got, ref_adj[k])
        assert fits[k]['rank'] == ref_fits[k]['rank']
        assert fits[k]['n_rows'] == ref_fits[k]['n_rows']
        if full_rank:
            close(fits[k]['coef'], ref_fits[k]['coef'])
            close(fits[k]['intercept'], ref_fits[k]['intercept'])
            close(fits[k]['singular'], ref_fits[k]['singular'])


def _shapes():
    out = []
    for N in NS:
        for q in QS:
            for p in PS:
                if q + p <= 256 and (N < 10 ** 6 or q <= 100 or p == 2):
                    out.append((N, q, p))
    return out


@pytest.mark.parametrize('N,q,p', _shapes())
def test_matches_restatement(N, q, p):
    rs = np.random.RandomState(N * 7 + q * 3 + p)
    S = summaries(N, q, rs)
    T = thetas(S, p, rs)
    o = S.mean(axis=0) + rs.randn(q) * S.std(axis=0) * 0.1
    # strided device views: S in a wider matrix, theta as a column slice
    wide = torch.zeros((N, q + 3), dtype=torch.float64, device='cuda')
    wide[:, 2:2 + q] = torch.from_numpy(S).cuda()
    Tw = torch.zeros((N, p + 1), dtype=torch.float64, device='cuda')
    Tw[:, 1:] = torch.from_numpy(T).cuda()
    adjusted, fits = ops.linear_adjust(wide[:, 2:2 + q], Tw[:, 1:], o)
    check(S, T, o, adjusted, fits, full_rank=N > q + 1)


def test_column_lists_and_host_input():
    rs = np.random.RandomState(1)
    S = summaries(3000, 5, rs)
    T = thetas(S, 3, rs)
    o = rs.randn(5)
    adjusted, fits = ops.linear_adjust([torch.from_numpy(c.copy()).cuda() for c in S.T],
                                       list(T.T), o)
    check(S, T, o, adjusted, fits)


@pytest.mark.parametrize('N', [257, 5000, 70000])
def test_masks_in_every_position(N):
    rs = np.random.RandomState(N)
    q, p = 4, 3
    S = summaries(N, q, rs)
    T = thetas(S, p, rs)
    o = rs.randn(q)
    edges = [0, 1, 31, 32, 255, 256, 2047, 2048, N - 1]
    pos = sorted({e for e in edges if e < N} | set(rs.randint(0, N, 20)))
    for i, r in enumerate(pos):
        if i % 3 == 0:
            S[r, i % q] = (np.nan, np.inf, -np.inf)[(i // 3) % 3]
        if i % 3 == 1:
            T[r, 1] = np.nan
        if i % 3 == 2:
            T[r, 2] = np.inf
            S[(r + 1) % N, 0] = np.nan
    adjusted, fits = ops.linear_adjust(S, T, o)
    check(S, T, o, adjusted, fits)
    assert len({f['n_rows'] for f in fits}) == 3


def test_nonfinite_observed_drops_everything():
    rs = np.random.RandomState(2)
    S = summaries(100, 2, rs)
    with pytest.raises(ValueError, match='n_samples = 0'):
        ops.linear_adjust(S, thetas(S, 1, rs), [0.0, np.nan])


def test_single_row_group():
    rs = np.random.RandomState(3)
    S = summaries(600, 3, rs)
    T = thetas(S, 2, rs)
    S[1:, 0] = np.nan
    adjusted, fits = ops.linear_adjust(S, T, np.zeros(3))
    for k in range(2):
        assert fits[k]['n_rows'] == 1 and fits[k]['rank'] == 0
        assert np.all(fits[k]['coef'] == 0)
        np.testing.assert_array_equal(adjusted[k].cpu().numpy(), T[:1, k])


def test_all_dropped_group_raises():
    rs = np.random.RandomState(4)
    S = summaries(600, 3, rs)
    T = thetas(S, 2, rs)
    T[:, 1] = np.nan
    with pytest.raises(ValueError, match='n_samples = 0'):
        ops.linear_adjust(S, T, np.zeros(3))


def test_limits():
    with pytest.raises(ValueError, match='q \\+ p <= 256'):
        ops.linear_adjust(np.zeros((4, 250)), np.zeros((4, 7)), np.zeros(250))
    with pytest.raises(ValueError, match='2\\^31'):
        ops.linear_adjust([np.broadcast_to(0.0, (2 ** 31,))], [np.broadcast_to(0.0, (2 ** 31,))],
                          [0.0])
    with pytest.raises(ValueError, match='1-d'):
        ops.linear_adjust([np.zeros((4, 2))], [np.zeros(4)], [0.0])


def test_bitwise_repeatable():
    rs = np.random.RandomState(5)
    S = summaries(300000, 40, rs)
    T = thetas(S, 6, rs)
    T[::977, 3] = np.nan
    o = rs.randn(40)
    Sd, Td = torch.from_numpy(S).cuda(), torch.from_numpy(T).cuda()
    a1, f1 = ops.linear_adjust(Sd, Td, o)
    for _ in range(2):
        a2, f2 = ops.linear_adjust(Sd, Td, o)
        for k in range(6):
            assert torch.equal(a1[k], a2[k])
            np.testing.assert_array_equal(f1[k]['coef'], f2[k]['coef'])
            assert f1[k]['intercept'] == f2[k]['intercept']


def _cases():
    from conftest import load_golden
    return [str(c) for c in load_golden('post_processing')['cases']]


@pytest.mark.parametrize('name', _cases())
def test_goldens(golden, name):
    g = golden('post_processing')
    sample, model, snames, pnames = case(g, name)
    adj = LinearAdjustment()
    if int(g[name + '_warned']):
        with pytest.warns(UserWarning, match='Non-finite'):
            adj.fit(sample, model, snames, pnames)
    else:
        adj.fit(sample, model, snames, pnames)
    res = adj.adjust()
    assert isinstance(res.outputs, results.DeviceOutputs)
    check_case(g, name, res.outputs, adj.regression_models)


def _gauss_model(seed=20170616, n_obs=50, mu=5, sigma=1, mu0=10, sigma0=100):
    y_obs = gauss.gauss(mu, sigma, n_obs=n_obs, batch_size=1,
                        random_state=np.random.RandomState(seed))
    m = elfi.ElfiModel()
    elfi.Prior('norm', mu0, sigma0, model=m, name='mu')
    elfi.Simulator(partial(gauss.gauss, sigma=sigma, n_obs=n_obs), m['mu'], observed=y_obs,
                   name='gauss')
    elfi.Summary(lambda x: x.mean(axis=1), m['gauss'], name='ss_mean')
    elfi.Distance('euclidean', m['ss_mean'], name='d')
    n = y_obs.shape[1]
    mu1 = (mu0 / sigma0 ** 2 + y_obs.sum() / sigma ** 2) / (1 / sigma0 ** 2 + n / sigma ** 2)
    sigma1 = (1 / sigma0 ** 2 + n / sigma ** 2) ** (-0.5)
    return m, mu1, sigma1


def test_reference_single_parameter(golden):
    g = golden('post_processing')
    m, _, _ = _gauss_model()
    res = elfi.Rejection(m['d'], output_names=['ss_mean'], batch_size=1000,
                         seed=20170616).sample(1000, threshold=1)
    np.testing.assert_array_equal(res.outputs['mu'], g['gauss_mu'])
    np.testing.assert_array_equal(res.outputs['ss_mean'], g['gauss_ss_mean'])
    adj = elfi.adjust_posterior(model=m, sample=res, parameter_names=['mu'],
                                summary_names=['ss_mean'])
    close(adj.outputs['mu'], g['gauss_adj_mu'])
    assert np.allclose(statistics(adj.outputs['mu']), (4.9772879640569778, 0.02058680115402544))


def test_reference_nonfinite_values(golden):
    g = golden('post_processing')
    m, _, _ = _gauss_model()
    res = elfi.Rejection(m['d'], output_names=['ss_mean'], batch_size=1000,
                         seed=20170616).sample(1000, threshold=1)
    np.testing.assert_array_equal(res.outputs['mu'], g['gauss_mu'])
    out = {'mu': np.append(res.outputs['mu'], np.inf),
           'ss_mean': np.append(res.outputs['ss_mean'], np.inf)}
    host = results.Sample(method_name='Rejection', outputs=out, parameter_names=['mu'])
    with pytest.warns(UserWarning):
        adj = elfi.adjust_posterior(model=m, sample=host, parameter_names=['mu'],
                                    summary_names=['ss_mean'])
    close(adj.outputs['mu'], g['gauss_adj_mu'])
    assert np.allclose(statistics(adj.outputs['mu']), (4.9772879640569778, 0.02058680115402544))


def test_reference_multi_parameter(golden):
    g = golden('post_processing')
    m = ma2.get_model(true_params=[0.6, 0.2], seed_obs=20170511)
    res = elfi.Rejection(m['d'], batch_size=1000, output_names=['S1', 'S2'],
                         seed=20170511).sample(500, threshold=0.2)
    for name in ('t1', 't2', 'S1', 'S2'):
        np.testing.assert_array_equal(res.outputs[name], g['ma2_' + name])
    adj = adjust_posterior(model=m, sample=res, parameter_names=['t1', 't2'],
                           summary_names=['S1', 'S2'], adjustment=LinearAdjustment())
    close(adj.outputs['t1'], g['ma2_adj_t1'])
    close(adj.outputs['t2'], g['ma2_adj_t2'])
    assert np.allclose(statistics(adj.outputs['t1']), (0.51606048286584782, 0.017253007645871756))
    assert np.allclose(statistics(adj.outputs['t2']), (0.15805189695581101, 0.028004406914362647))


def test_conjugate_gaussian_posterior():
    m, mu1, sigma1 = _gauss_model()
    n = 20000
    res = elfi.Rejection(m['d'], output_names=['ss_mean'], batch_size=100000,
                         seed=7).sample(n, threshold=1)
    adj = elfi.adjust_posterior(res, m, ['ss_mean'], ['mu'])
    a = adj.outputs['mu']
    assert len(a) == n
    se_mean = sigma1 / np.sqrt(n)
    se_var = sigma1 ** 2 * np.sqrt(2.0 / (n - 1))
    assert abs(a.mean() - mu1) <= 4 * se_mean, (a.mean(), mu1, se_mean)
    assert abs(a.var() - sigma1 ** 2) <= 4 * se_var, (a.var(), sigma1 ** 2, se_var)


def test_device_ma2_million_rows():
    m = ma2.get_device_model(true_params=[0.6, 0.2], seed_obs=3)
    res = elfi.Rejection(m['d'], output_names=['S1', 'S2'], batch_size=10 ** 6,
                         seed=11).sample(10 ** 6, quantile=0.1, bar=False)
    assert isinstance(res.outputs, results.DeviceOutputs)
    adj = adjust_posterior(res, m, ['S1', 'S2'])
    assert isinstance(adj.outputs, results.DeviceOutputs)
    S = np.column_stack([res.outputs['S1'], res.outputs['S2']])
    T = np.column_stack([res.outputs['t1'], res.outputs['t2']])
    from elfi_b200.post_processing import _observed
    ref, _ = ld.linear_adjust(S, T, _observed(m, ['S1', 'S2']))
    assert len(ref[0]) == 10 ** 6
    close(adj.outputs['t1'], ref[0])
    close(adj.outputs['t2'], ref[1])
