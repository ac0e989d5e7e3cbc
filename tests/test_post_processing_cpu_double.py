"""The unmodified regression-adjustment host module under the CPU double of the C ABI
(tests/linadjust_double.py) reproduces the reference's goldens, warning included."""
import warnings

import numpy as np
import pytest

import abi_double
import linadjust_double
from post_processing_cases import case, check_case, close, statistics
from elfi_b200 import adjust_posterior, results
from elfi_b200.post_processing import LinearAdjustment


def _cases():
    from conftest import load_golden
    return [str(c) for c in load_golden('post_processing')['cases']]


@pytest.mark.parametrize('name', _cases())
def test_goldens(cpu_double, monkeypatch, golden, name):
    abi_double.install(monkeypatch, linadjust_double.TABLE)
    g = golden('post_processing')
    sample, model, snames, pnames = case(g, name)
    adj = LinearAdjustment()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter('always')
        adj.fit(sample, model, snames, pnames)
    assert len(caught) == int(g[name + '_warned'])
    if caught:
        assert caught[0].category is UserWarning
        assert str(caught[0].message) == 'Non-finite inputs and outputs will be omitted.'
    res = adj.adjust()
    assert isinstance(res.outputs, results.DeviceOutputs)
    assert res.method_name == 'LinearAdjustment' and res.parameter_names == pnames
    check_case(g, name, res.outputs, adj.regression_models)
    np.testing.assert_array_equal(adj.X, np.column_stack([sample.outputs[s] for s in snames])
                                  - g[name + '_o'])
    assert cpu_double.CALLS.count('elfi_b200_regadj_mask_f64') == 1


def test_functional_goldens(cpu_double, monkeypatch, golden):
    abi_double.install(monkeypatch, linadjust_double.TABLE)
    from elfi_b200.examples import ma2
    g = golden('post_processing')
    m = ma2.get_model(true_params=[0.6, 0.2], seed_obs=20170511)
    out = {k: g['ma2_' + k] for k in ('t1', 't2', 'S1', 'S2')}
    res = results.Sample(method_name='Rejection', outputs=out, parameter_names=['t1', 't2'])
    adj = adjust_posterior(res, m, ['S1', 'S2'], ['t1', 't2'], adjustment=LinearAdjustment())
    close(adj.outputs['t1'], g['ma2_adj_t1'])
    close(adj.outputs['t2'], g['ma2_adj_t2'])
    assert np.allclose(statistics(adj.outputs['t1']), (0.51606048286584782, 0.017253007645871756))
    assert np.allclose(statistics(adj.outputs['t2']), (0.15805189695581101, 0.028004406914362647))


def test_all_dropped_raises(cpu_double, monkeypatch, golden):
    abi_double.install(monkeypatch, linadjust_double.TABLE)
    sample, model, snames, pnames = case(golden('post_processing'), 'q2p3')
    sample.outputs['t1'] = np.full_like(sample.outputs['t1'], np.nan)
    with pytest.raises(ValueError, match='n_samples = 0'):
        adjust_posterior(sample, model, snames, pnames)
