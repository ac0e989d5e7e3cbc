"""Bayesian synthetic likelihood on the host: the NumPy restatement of the device likelihood
against the reference's pdf_methods, the logit transform of the proposals, and argument errors."""
import numpy as np
import pytest

import abi_double
import bsl_double
from elfi_b200 import bsl, ops
from elfi_b200.examples import ma2


def _close(a, b, rel=1e-10):
    a, b = np.asarray(a, dtype=float), np.asarray(b, dtype=float)
    assert a.shape == b.shape
    assert np.array_equal(np.isneginf(a), np.isneginf(b)), (a, b)
    f = np.isfinite(b)
    assert np.all(np.abs(a[f] - b[f]) <= rel * (1 + np.abs(b[f]))), (a, b)


def test_oracle_matches_reference_likelihoods(golden):
    g = golden('bsl_pdf')
    ssx, ssy = g['ssx'], g['ssy']
    _close(bsl_double.synlik(ssx, ssy), g['standard'])
    _close(bsl_double.synlik(ssx, ssy, penalties=g['penalties'])[0], g['warton'])
    _close(bsl_double.synlik(ssx, ssy, W=g['W']), g['whitened'])
    _close(bsl_double.synlik(ssx, ssy, penalties=[0.35], W=g['W'])[0], g['whitened_warton'])
    _close(bsl_double.synlik(ssx, ssy, 'unbiased'), g['unbiased'])
    _close(bsl_double.synlik(g['ssx_dup'], ssy), g['dup'])
    _close(bsl_double.synlik(g['ssx_const'], ssy), g['const'])
    _close(bsl_double.synlik(g['ssx_d1'], g['ssy_d1']), g['d1'])
    assert np.isneginf(g['dup'][0]) and np.isneginf(g['const'][0])


def test_oracle_non_finite_group_only():
    rs = np.random.RandomState(1)
    S = rs.randn(3, 40, 4)
    S[1, 7, 2] = np.nan
    ll = bsl_double.synlik(S, np.zeros(4))
    assert np.isneginf(ll[1]) and np.all(np.isfinite(ll[[0, 2]]))


def test_logit_transform_matches_reference(golden):
    g = golden('bsl_pdf')
    bound = g['logit_bound']
    with np.errstate(all='ignore'):
        for x, t, back, jac in zip(g['logit_points'], g['logit'], g['logit_back'], g['logit_jac']):
            np.testing.assert_array_equal(bsl.BSL._para_logit_transform(x, bound), t)
            np.testing.assert_array_equal(bsl.BSL._para_logit_back_transform(t, bound), back)
            assert bsl.BSL._jacobian_logit_transform(x, bound) == jac


def test_likelihood_argument_errors():
    with pytest.raises(ValueError):
        bsl.standard_likelihood(shrinkage='warton', penalty=1.5)
    with pytest.raises(ValueError):
        bsl.standard_likelihood(shrinkage='warton', penalty=-0.1)
    with pytest.raises(ValueError):
        bsl.standard_likelihood(shrinkage='warton')
    with pytest.raises(NotImplementedError, match='glasso'):
        bsl.standard_likelihood(shrinkage='glasso', penalty=0.1)
    with pytest.raises(NotImplementedError, match='semiBSL'):
        bsl.semiparametric_likelihood()
    with pytest.raises(NotImplementedError, match='R-BSL'):
        bsl.robust_likelihood('mean')


def test_pre_sample_tool_errors():
    m = ma2.get_model(n_obs=10, seed_obs=4)
    with pytest.raises(NotImplementedError, match='glasso'):
        bsl.select_penalty(m, 50, [.6, .2], ['MA2'])
    with pytest.raises(NotImplementedError, match='semiBSL'):
        bsl.estimate_whitening_matrix(m, 50, [.6, .2], ['MA2'], likelihood_type='semiparametric')
    with pytest.raises(ValueError):
        bsl.estimate_whitening_matrix(m, 50, [.6, .2], ['MA2'], likelihood_type='other')


def test_bsl_argument_errors():
    m = ma2.get_model(n_obs=10, seed_obs=4)
    with pytest.raises(ValueError, match='multiple of batch_size'):
        bsl.BSL(m, 100, ['MA2'], batch_size=30)
    with pytest.raises(ValueError, match='not found'):
        bsl.BSL(m, 100, ['nope'])
    big = ma2.get_model(n_obs=161, seed_obs=4)
    with pytest.raises(ValueError, match='160'):
        bsl.BSL(big, 100, ['MA2'])


def test_synlik_argument_errors(cpu_double, monkeypatch):
    abi_double.install(monkeypatch, bsl_double.TABLE)
    rs = np.random.RandomState(2)
    S, y = rs.randn(20, 3), np.zeros(3)
    with pytest.raises(ValueError, match=r'\[0, 1\]'):
        ops.synlik(S, y, penalties=[0.2, 1.2])
    with pytest.raises(ValueError, match='160'):
        ops.synlik(rs.randn(200, 161), np.zeros(161))
    with pytest.raises(ValueError, match='n >= 2'):
        ops.synlik(S[:1], y)
    with pytest.raises(ValueError, match='unbiased'):
        ops.synlik(S, y, estimator='unbiased', penalties=[0.1])
    with pytest.raises(ValueError, match='unbiased'):
        ops.synlik(S, y, estimator='unbiased', whitening=np.eye(3))
    with pytest.raises(ValueError, match='estimator'):
        ops.synlik(S, y, estimator='semiparametric')
    with pytest.raises(ValueError, match='y has'):
        ops.synlik(S, np.zeros(4))
    with pytest.raises(ValueError, match='whitening'):
        ops.synlik(S, y, whitening=np.eye(4))
    ll = ops.synlik(S, y, penalties=[0.0, 0.5])
    assert tuple(ll.shape) == (1, 2)
    np.testing.assert_array_equal(ll.cpu().numpy(), bsl_double.synlik(S, y, penalties=[0.0, 0.5]))
