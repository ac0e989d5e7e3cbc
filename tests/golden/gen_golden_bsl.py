"""Golden fixtures for Bayesian synthetic likelihood, from the UNMODIFIED reference (elfi-dev/elfi,
the checkout named by ELFI_REFERENCE_ROOT).

    ELFI_REFERENCE_ROOT=<checkout> python tests/golden/gen_golden_bsl.py

* bsl_pdf.npz    -- gaussian_syn_likelihood and gaussian_syn_likelihood_ghurye_olkin on crafted
                    summaries: standard; Warton at several penalties; whitening, alone and with a
                    penalty; unbiased; a duplicated and a constant column (-inf); d = 1.  Also
                    the logit transform, its inverse and its Jacobian for each kind of bound.
* bsl_chains.npz -- BSL chains on ma2.get_model(n_obs=50, true_params=[.6, .2], seed_obs=4) with
                    feature MA2 (d = 50), n_sim_round = 500, seed = 123, params0 = [.6, .2],
                    200 iterations: standard, unbiased, standard with burn_in and
                    logit_transform_bound, whitened Warton.  Each chain: samples_all,
                    state['logposterior'], acc_rate, n_sim.  With them the whitening matrix
                    estimate_whitening_matrix(m, 5000, [.6, .2], ['MA2'], seed=1) and
                    select_penalty(m, 100, [.6, .2], ['MA2'], M=10, shrinkage='warton',
                    whitening=W, seed=1).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

from ref_shim import import_reference  # noqa: E402

elfi = import_reference()
from elfi.examples import ma2  # noqa: E402
from elfi.methods.bsl import pdf_methods as pm  # noqa: E402
from elfi.methods.bsl.pre_sample_methods import (estimate_whitening_matrix,  # noqa: E402
                                                 select_penalty)

CHAIN = dict(n_sim_round=500, seed=123, params0=[.6, .2], n_iter=200,
             sigma=[[.02, .01], [.01, .02]])
PENALTIES = [0.0, 0.1, 0.35, 0.7, 1.0]
BOUND = np.array([[-2., 2.], [-np.inf, 1.], [0., np.inf], [-np.inf, np.inf]])
LOGIT_POINTS = np.array([[-1.5, 0.3, 0.2, -3.], [0.4, -7., 5., 2.5], [1.99, 0.999, 1e-3, 0.]])


def save(name, **arrays):
    np.savez(os.path.join(HERE, name + '.npz'), **arrays)
    print('wrote', name, {k: np.shape(v) for k, v in arrays.items()})


def pdf_cases():
    rs = np.random.RandomState(0)
    d = 6
    A = rs.randn(d, d) * 0.5 + np.eye(d)
    ssx = rs.randn(300, d) @ A + rs.randn(d)
    ssy = ssx.mean(axis=0) + 0.3 * rs.randn(d)
    W = np.eye(d) + 0.2 * rs.randn(d, d)
    out = dict(ssx=ssx, ssy=ssy, W=W, penalties=np.array(PENALTIES))
    out['standard'] = pm.gaussian_syn_likelihood(ssx, ssy)
    out['warton'] = np.concatenate([pm.gaussian_syn_likelihood(ssx, ssy, shrinkage='warton',
                                                                penalty=p) for p in PENALTIES])
    out['whitened'] = pm.gaussian_syn_likelihood(ssx, ssy, whitening=W)
    out['whitened_warton'] = pm.gaussian_syn_likelihood(ssx, ssy, shrinkage='warton', penalty=0.35,
                                                        whitening=W)
    out['unbiased'] = pm.gaussian_syn_likelihood_ghurye_olkin(ssx, ssy)
    dup = ssx.copy()
    dup[:, 4] = dup[:, 1]
    const = ssx.copy()
    const[:, 2] = 1.5
    out['ssx_dup'], out['ssx_const'] = dup, const
    out['dup'] = pm.gaussian_syn_likelihood(dup, ssy)
    out['const'] = pm.gaussian_syn_likelihood(const, ssy)
    ssx1 = rs.randn(50, 1) * 2 + 1
    out['ssx_d1'], out['ssy_d1'] = ssx1, np.array([0.5])
    out['d1'] = pm.gaussian_syn_likelihood(ssx1, np.array([0.5]))
    BSL = elfi.BSL
    out['logit_bound'] = BOUND
    out['logit_points'] = LOGIT_POINTS
    with np.errstate(all='ignore'):
        out['logit'] = np.array([BSL._para_logit_transform(x, BOUND) for x in LOGIT_POINTS])
        out['logit_back'] = np.array([BSL._para_logit_back_transform(t, BOUND)
                                      for t in out['logit']])
        out['logit_jac'] = np.array([BSL._jacobian_logit_transform(x, BOUND)
                                     for x in LOGIT_POINTS])
    return out


def chain(likelihood, **sample_kw):
    m = ma2.get_model(n_obs=50, true_params=[.6, .2], seed_obs=4)
    bsl = elfi.BSL(m, CHAIN['n_sim_round'], ['MA2'], likelihood=likelihood, seed=CHAIN['seed'])
    res = bsl.sample(CHAIN['n_iter'], sigma_proposals=np.array(CHAIN['sigma']),
                     params0=np.array(CHAIN['params0']), **sample_kw)
    return dict(samples_all=np.column_stack([res.samples_all[p] for p in ['t1', 't2']]),
                logposterior=np.array(bsl.state['logposterior']), acc_rate=np.float64(res.acc_rate),
                n_sim=np.int64(res.n_sim))


def chains():
    m = ma2.get_model(n_obs=50, true_params=[.6, .2], seed_obs=4)
    W = estimate_whitening_matrix(m, 5000, np.array([.6, .2]), ['MA2'], seed=1)
    pen, std = select_penalty(model=m, n_sim=100, theta=np.array([.6, .2]), feature_names=['MA2'],
                              M=10, shrinkage='warton', whitening=W, sigma=1.5, seed=1)
    out = dict(W=W, penalty=pen, penalty_std=std)
    runs = {
        'standard': (None, {}),
        'unbiased': (pm.unbiased_likelihood(), {}),
        'bounded': (None, dict(burn_in=50, logit_transform_bound=[[-2., 2.], [-1., 1.]])),
        'whitened': (pm.standard_likelihood(shrinkage='warton', penalty=pen, whitening=W), {}),
    }
    for name, (lik, kw) in runs.items():
        for k, v in chain(lik, **kw).items():
            out[name + '_' + k] = v
    return out


if __name__ == '__main__':
    save('bsl_pdf', **pdf_cases())
    save('bsl_chains', **chains())
