"""Golden fixtures for the regression adjustment, from the UNMODIFIED reference (elfi-dev/elfi, the
checkout named by ELFI_REFERENCE_ROOT), whose LinearAdjustment fits scikit-learn's
LinearRegression.  Written with scikit-learn 1.9.0, NumPy 2.3.5 and SciPy 1.18.1.

    ELFI_REFERENCE_ROOT=<checkout> python tests/golden/gen_golden_post_processing.py

post_processing.npz holds, for each crafted case <c> (names in `cases`):
  <c>_S (N, q), <c>_T (N, p), <c>_o (q,)  the summaries, parameters and observed summaries;
  <c>_pidx                                 the columns of T passed as parameter_names, in order;
  <c>_warned                               1 if the reference warned about non-finite rows;
  <c>_adj<i>, <c>_coef<i>, <c>_intercept<i>, <c>_rank<i>  for the i-th adjusted parameter.
and for the reference's functional tests (tests/functional/test_post_processing.py):
  gauss_mu, gauss_ss_mean, gauss_adj_mu    Rejection outputs and the adjusted mu;
  ma2_t1, ma2_t2, ma2_S1, ma2_S2, ma2_adj_t1, ma2_adj_t2.
"""
import os
import sys
import types
import warnings
from functools import partial

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

from ref_shim import import_reference  # noqa: E402

elfi = import_reference()
from elfi.examples import gauss, ma2  # noqa: E402
from elfi.methods import results  # noqa: E402
from elfi.methods.post_processing import LinearAdjustment, adjust_posterior  # noqa: E402


def conditioned(rs, N, q, cond=30.0):
    """(N, q) summaries with a moderate condition number."""
    Q, _ = np.linalg.qr(rs.randn(N, q))
    rot, _ = np.linalg.qr(rs.randn(q, q))
    return (Q * np.geomspace(1.0, cond, q)) @ rot * np.sqrt(N) + rs.randn(q)


def response(rs, S, p):
    B = rs.randn(S.shape[1], p)
    return S @ B * 0.1 + rs.randn(p) + 0.3 * rs.randn(S.shape[0], p)


def crafted():
    rs = np.random.RandomState(20261017)
    cases = {}
    for q in (1, 2, 6, 20):
        for p in (1, 3):
            S = conditioned(rs, 400, q)
            cases['q{}p{}'.format(q, p)] = (S, response(rs, S, p), rs.randn(q), list(range(p)))
    S = conditioned(rs, 300, 6)
    T = response(rs, S, 3)
    o = rs.randn(6)
    Sn = S.copy()
    Sn[[3, 50, 299], [0, 2, 5]] = [np.nan, np.inf, -np.inf]
    cases['nonfinite_S'] = (Sn, T, o, [0, 1, 2])
    Tn = T.copy()
    Tn[[7, 8, 120], 1] = [np.nan, np.inf, np.nan]
    cases['nonfinite_theta'] = (S, Tn, o, [0, 1, 2])
    Tb = Tn.copy()
    Tb[[0, 200], 2] = np.inf
    cases['nonfinite_both'] = (Sn, Tb, o, [0, 1, 2])
    base = conditioned(rs, 250, 4)
    cases['duplicate'] = (np.column_stack([base, base[:, 1]]), response(rs, base, 2),
                          rs.randn(5), [0, 1])
    cases['constant'] = (np.column_stack([base[:, :2], np.full(250, 1.5), base[:, 2:]]),
                         response(rs, base, 2), rs.randn(5), [0, 1])
    cases['sum_constant'] = (np.column_stack([base, 3.0 - base[:, 0]]), response(rs, base, 2),
                             rs.randn(5), [0, 1])
    S = conditioned(rs, 300, 3)
    cases['subset'] = (S, response(rs, S, 4), rs.randn(3), [3, 1])
    return cases


def run_case(S, T, o, pidx):
    names = ['s{}'.format(j) for j in range(S.shape[1])]
    pnames = ['t{}'.format(k) for k in range(T.shape[1])]
    outputs = dict(zip(names, S.T))
    outputs.update(zip(pnames, T.T))
    sample = results.Sample(method_name='crafted', outputs=outputs, parameter_names=pnames)
    model = {s: types.SimpleNamespace(observed=np.array([v])) for s, v in zip(names, o)}
    adj = LinearAdjustment()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter('always')
        adj.fit(sample, model, names, [pnames[k] for k in pidx])
    out = adj.adjust()
    res = dict(warned=np.int64(len(caught) > 0))
    for i, k in enumerate(pidx):
        m = adj.regression_models[i]
        res['adj{}'.format(i)] = out.outputs[pnames[k]]
        res['coef{}'.format(i)] = m.coef_
        res['intercept{}'.format(i)] = np.float64(m.intercept_)
        res['rank{}'.format(i)] = np.int64(m.rank_)
    return res


def functional():
    out = {}
    seed, n_obs, mu, sigma, mu0, sigma0 = 20170616, 50, 5, 1, 10, 100
    y_obs = gauss.gauss(mu, sigma, n_obs=n_obs, batch_size=1,
                        random_state=np.random.RandomState(seed))
    m = elfi.ElfiModel()
    elfi.Prior('norm', mu0, sigma0, model=m, name='mu')
    elfi.Simulator(partial(gauss.gauss, sigma=sigma, n_obs=n_obs), m['mu'], observed=y_obs,
                   name='gauss')
    elfi.Summary(lambda x: x.mean(axis=1), m['gauss'], name='ss_mean')
    elfi.Distance('euclidean', m['ss_mean'], name='d')
    res = elfi.Rejection(m['d'], output_names=['ss_mean'], batch_size=1000,
                         seed=seed).sample(1000, threshold=1)
    out['gauss_mu'] = res.outputs['mu']
    out['gauss_ss_mean'] = res.outputs['ss_mean']
    adj = elfi.adjust_posterior(model=m, sample=res, parameter_names=['mu'],
                                summary_names=['ss_mean'])
    out['gauss_adj_mu'] = adj.outputs['mu']

    seed = 20170511
    m = ma2.get_model(true_params=[0.6, 0.2], seed_obs=seed)
    res = elfi.Rejection(m['d'], batch_size=1000, output_names=['S1', 'S2'],
                         seed=seed).sample(500, threshold=0.2)
    for name in ('t1', 't2', 'S1', 'S2'):
        out['ma2_' + name] = res.outputs[name]
    adj = adjust_posterior(model=m, sample=res, parameter_names=['t1', 't2'],
                           summary_names=['S1', 'S2'], adjustment=LinearAdjustment())
    out['ma2_adj_t1'] = adj.outputs['t1']
    out['ma2_adj_t2'] = adj.outputs['t2']
    return out


def main():
    arrays = {}
    cases = crafted()
    arrays['cases'] = np.array(sorted(cases))
    for name, (S, T, o, pidx) in sorted(cases.items()):
        arrays[name + '_S'], arrays[name + '_T'], arrays[name + '_o'] = S, T, o
        arrays[name + '_pidx'] = np.array(pidx, dtype=np.int64)
        for k, v in run_case(S, T, o, pidx).items():
            arrays[name + '_' + k] = v
    arrays.update(functional())
    np.savez_compressed(os.path.join(HERE, 'post_processing.npz'), **arrays)
    print('wrote post_processing', len(arrays), 'arrays')


if __name__ == '__main__':
    main()
