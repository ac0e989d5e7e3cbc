"""Regression adjustment without a GPU: the NumPy restatement of the device path
(tests/linadjust_double.py) against the reference's goldens, and the host module's errors, options
and host path (tests/golden/gen_golden_post_processing.py)."""
import types

import numpy as np
import pytest

import linadjust_double as ld
from post_processing_cases import RANK_DEFICIENT, case, close
from elfi_b200 import post_processing as pp
from elfi_b200 import results
from elfi_b200.post_processing import LinearAdjustment, RegressionAdjustment, adjust_posterior


def _cases():
    from conftest import load_golden
    return [str(c) for c in load_golden('post_processing')['cases']]


@pytest.mark.parametrize('name', _cases())
def test_restatement_matches_reference(golden, name):
    g = golden('post_processing')
    T = g[name + '_T']
    pidx = list(g[name + '_pidx'])
    adjusted, fits = ld.linear_adjust(g[name + '_S'], T[:, pidx], g[name + '_o'])
    for i, fit in enumerate(fits):
        key = '{}_{{}}{}'.format(name, i)
        close(adjusted[i], g[key.format('adj')])
        assert fit['rank'] == int(g[key.format('rank')])
        if name not in RANK_DEFICIENT:
            close(fit['coef'], g[key.format('coef')])
            close(fit['intercept'], g[key.format('intercept')])


def test_restatement_functional_goldens(cpu_double, golden):
    g = golden('post_processing')
    adj, _ = ld.linear_adjust(np.column_stack([g['ma2_S1'], g['ma2_S2']]),
                              np.column_stack([g['ma2_t1'], g['ma2_t2']]),
                              _ma2_observed())
    close(adj[0], g['ma2_adj_t1'])
    close(adj[1], g['ma2_adj_t2'])


def _ma2_observed():
    from elfi_b200.examples import ma2
    m = ma2.get_model(true_params=[0.6, 0.2], seed_obs=20170511)
    return pp._observed(m, ['S1', 'S2'])


def test_get_adjustment():
    with pytest.raises(ValueError):
        pp._get_adjustment('doesnotexist')
    adj = LinearAdjustment()
    assert pp._get_adjustment(adj) is adj
    assert isinstance(pp._get_adjustment('linear'), LinearAdjustment)


@pytest.mark.parametrize('attr', ['X', 'sample', 'parameter_names'])
def test_attributes_before_fit(attr):
    with pytest.raises(ValueError, match='fitted first'):
        getattr(LinearAdjustment(), attr)


def test_missing_summary(golden):
    sample, model, snames, pnames = case(golden('post_processing'), 'q2p1')
    with pytest.raises(KeyError):
        adjust_posterior(sample, model, snames + ['nope'], pnames)


def test_non_scalar_parameter_and_2d_summary(cpu_double, golden):
    sample, model, snames, pnames = case(golden('post_processing'), 'q2p1')
    sample.outputs['t0'] = np.column_stack([sample.outputs['t0']] * 2)
    with pytest.raises(ValueError, match='1-d'):
        adjust_posterior(sample, model, snames, pnames)
    sample, model, snames, pnames = case(golden('post_processing'), 'q2p1')
    sample.outputs['s1'] = np.column_stack([sample.outputs['s1']] * 2)
    model['s1'] = types.SimpleNamespace(observed=np.array([[0.1]]))
    with pytest.raises(ValueError, match='1-d'):
        adjust_posterior(sample, model, snames, pnames)


@pytest.mark.parametrize('kw', [dict(fit_intercept=False), dict(positive=True)])
def test_unsupported_options(kw):
    with pytest.raises(NotImplementedError, match=list(kw)[0]):
        LinearAdjustment(**kw)


def test_ignored_options_accepted():
    LinearAdjustment(copy_X=False, n_jobs=4, tol=1e-8)


class NumpyLstsq:
    """A host regression model: least squares with an intercept through NumPy."""

    def fit(self, X, y):
        Z = np.column_stack([np.ones(len(X)), X])
        beta = np.linalg.lstsq(Z, y, rcond=None)[0]
        self.intercept_, self.coef_ = beta[0], beta[1:]
        return self


class HostAdjustment(RegressionAdjustment):
    _regression_model = NumpyLstsq
    _name = 'HostAdjustment'

    def _adjust(self, i, theta_i, regression_model):
        return theta_i - self.X[self._finite[i], :] @ regression_model.coef_

    def _input_variables(self, model, sample, summary_names):
        S = np.stack([sample.outputs[s] for s in summary_names], axis=1)
        return S - np.array([model[s].observed[0] for s in summary_names])


def test_host_subclass(golden):
    g = golden('post_processing')
    sample, model, snames, pnames = case(g, 'nonfinite_both')
    with pytest.warns(UserWarning, match='Non-finite'):
        res = adjust_posterior(sample, model, snames, pnames, adjustment=HostAdjustment())
    assert res.method_name == 'HostAdjustment'
    assert isinstance(res, results.Sample) and not isinstance(res.outputs, results.DeviceOutputs)
    for i, pn in enumerate(pnames):
        close(res.outputs[pn], g['nonfinite_both_adj{}'.format(i)])
