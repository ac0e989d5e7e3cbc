"""Shared helpers of the regression-adjustment tests: golden cases as samples and models."""
import types

import numpy as np

from elfi_b200 import results

RANK_DEFICIENT = ('duplicate', 'constant', 'sum_constant')


def close(got, ref, tol=1e-9):
    got, ref = np.asarray(got, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    err = np.abs(got - ref) / (1 + np.abs(ref))
    assert np.all(err <= tol), float(np.max(err))


def case(g, name):
    """(sample, model, summary names, parameter names) of golden case `name`, host outputs."""
    S, T, o = g[name + '_S'], g[name + '_T'], g[name + '_o']
    snames = ['s{}'.format(j) for j in range(S.shape[1])]
    pnames = ['t{}'.format(k) for k in range(T.shape[1])]
    outputs = dict(zip(snames, S.T.copy()))
    outputs.update(zip(pnames, T.T.copy()))
    sample = results.Sample(method_name='crafted', outputs=outputs, parameter_names=pnames)
    model = {s: types.SimpleNamespace(observed=np.array([v])) for s, v in zip(snames, o)}
    return sample, model, snames, [pnames[k] for k in g[name + '_pidx']]


def check_case(g, name, adjusted, models):
    """adjusted (name -> column) and the fitted models against golden case `name`."""
    _, _, _, pnames = case(g, name)
    for i, pn in enumerate(pnames):
        key = '{}_{{}}{}'.format(name, i)
        close(adjusted[pn], g[key.format('adj')])
        assert models[i].rank_ == int(g[key.format('rank')])
        if name not in RANK_DEFICIENT:
            close(models[i].coef_, g[key.format('coef')])
            close(models[i].intercept_, g[key.format('intercept')])


def statistics(a):
    return a.mean(), a.var()
