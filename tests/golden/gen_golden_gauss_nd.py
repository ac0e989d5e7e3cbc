"""Golden fixtures for the n-D Gaussian mean model (gauss.get_model(nd_mean=True)), from the
UNMODIFIED reference (elfi-dev/elfi, the checkout named by ELFI_REFERENCE_ROOT).

    ELFI_REFERENCE_ROOT=<checkout> python tests/golden/gen_golden_gauss_nd.py

gauss_nd.npz holds, for each configuration <c> of CONFIGS (D = 1 with cov [1], D = 2 with
[[1, .5], [.5, 1]], D = 5 with cov_matrix=None):
* <c>_observed                  the model's observed data (1, n_obs, D);
* <c>_gen_<node>                m.generate(GENERATE_N, seed=GENERATE_SEED) for every mu_i, gauss,
                                ss_mean, ss_var and d;
* <c>_<run>_mu_<i>, _d, _n_sim, _threshold
                                Rejection in quantile, n_sim and threshold mode (REJECTION);
* <c>_smc_...                   SMC with two thresholds: the final samples, discrepancies,
                                weights and threshold, and per population pop<k>_ the same with
                                n_sim, and smc_n_pops.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

from ref_shim import import_reference  # noqa: E402

elfi = import_reference()
from elfi.examples import gauss  # noqa: E402

CONFIGS = {
    'd1': dict(true_params=[4], cov_matrix=[1], seed_obs=3, threshold=0.5, smc=[1.0, 0.5]),
    'd2': dict(true_params=[4, 4], cov_matrix=[[1, .5], [.5, 1]], seed_obs=4, threshold=1.0,
               smc=[2.0, 1.0]),
    'd5': dict(true_params=[1, 2, 3, 4, 5], cov_matrix=None, seed_obs=5, threshold=3.5,
               smc=[4.0, 3.0]),
}
GENERATE_N, GENERATE_SEED = 20, 11
REJECTION = {'quantile': (dict(batch_size=1000, seed=123), dict(n_samples=100, quantile=0.01)),
             'nsim': (dict(batch_size=500, seed=7), dict(n_samples=64, n_sim=3000)),
             'threshold': (dict(batch_size=1000, seed=123), dict(n_samples=150))}
SMC = (dict(batch_size=1000, seed=20), dict(n_samples=150))


def model(c):
    return gauss.get_model(true_params=c['true_params'], seed_obs=c['seed_obs'], nd_mean=True,
                           cov_matrix=c['cov_matrix'])


def run_arrays(prefix, res, names):
    out = {prefix + k: np.asarray(res.samples[k]) for k in names}
    out.update({prefix + 'd': np.asarray(res.discrepancies), prefix + 'n_sim': np.int64(res.n_sim),
                prefix + 'threshold': np.float64(res.threshold)})
    return out


def main():
    out = {}
    for tag, c in CONFIGS.items():
        m = model(c)
        names = ['mu_{}'.format(i) for i in range(len(c['true_params']))]
        out[tag + '_observed'] = np.asarray(m.observed['gauss'])
        gen = m.generate(GENERATE_N, seed=GENERATE_SEED)
        for k in names + ['gauss', 'ss_mean', 'ss_var', 'd']:
            out['{}_gen_{}'.format(tag, k)] = np.asarray(gen[k])
        for run, (init, kw) in REJECTION.items():
            kw = dict(kw, threshold=c['threshold']) if run == 'threshold' else kw
            res = elfi.Rejection(m['d'], **init).sample(bar=False, **kw)
            out.update(run_arrays('{}_{}_'.format(tag, run), res, names))
        res = elfi.SMC(m['d'], **SMC[0]).sample(bar=False, thresholds=c['smc'], **SMC[1])
        pre = tag + '_smc_'
        out.update(run_arrays(pre, res, names))
        out[pre + 'weights'] = np.asarray(res.weights)
        out[pre + 'n_pops'] = np.int64(len(res.populations))
        for i, pop in enumerate(res.populations):
            out.update(run_arrays('{}pop{}_'.format(pre, i), pop, names))
            out['{}pop{}_weights'.format(pre, i)] = np.asarray(pop.weights)
        print(tag, 'done')
    np.savez(os.path.join(HERE, 'gauss_nd.npz'), **out)
    print('wrote gauss_nd', {k: np.shape(v) for k, v in out.items()})


if __name__ == '__main__':
    main()
