"""Golden fixtures for the AR(1) example and compare_models, from the UNMODIFIED reference
(elfi-dev/elfi, the checkout named by ELFI_REFERENCE_ROOT).

    ELFI_REFERENCE_ROOT=<checkout> python tests/golden/gen_golden_ar1.py

* ar1_draws.npz      -- elfi.examples.ar1.AR1 for seeded RandomStates at batch 1 and 16, phi in
                        {-1, -0.5, 0, 0.9, 1} and n_obs in {1, 2, 200}: key phi{j}_n{n}_b{b}.
* ar1_rejection.npz  -- the reference's test_ar1 (Rejection(get_model()['d'], batch_size=10)
                        .sample(10, quantile=0.5)) with fixed seeds, and one quantile run with a
                        larger batch.
* compare_models.npz -- elfi.compare_models on the configuration of the reference's
                        test_compare_models (gauss; the same with a wider prior on mu through
                        become; an MA2 simulator), with fixed seeds: each sample's discrepancies,
                        n_samples and n_sim, and p with and without model priors.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

from ref_shim import import_reference  # noqa: E402

elfi = import_reference()
from elfi.examples import ar1, gauss, ma2  # noqa: E402

PHIS = (-1.0, -0.5, 0.0, 0.9, 1.0)
N_OBS = (1, 2, 200)
TEST_AR1 = dict(seed_obs=4, batch_size=10, seed=5, n=10, quantile=0.5)
QUANTILE = dict(seed_obs=1, batch_size=100, seed=3, n=50, quantile=0.1)
COMPARE = dict(seed_obs=6, n=100, seeds=(7, 8, 9))
MODEL_PRIORS = np.array([0.2, 0.3, 0.5])


def save(name, **arrays):
    np.savez(os.path.join(HERE, name + '.npz'), **arrays)
    print('wrote', name, {k: np.shape(v) for k, v in arrays.items()})


def rejection(a):
    m = ar1.get_model(seed_obs=a['seed_obs'])
    res = elfi.Rejection(m['d'], batch_size=a['batch_size'], seed=a['seed']).sample(
        a['n'], quantile=a['quantile'])
    return m, res


def main():
    out = dict(phis=np.array(PHIS))
    for j, phi in enumerate(PHIS):
        for n in N_OBS:
            for b in (1, 16):
                rs = np.random.RandomState(100 * j + 10 * n + b)
                out['phi{}_n{}_b{}'.format(j, n, b)] = ar1.AR1(phi, n_obs=n, batch_size=b,
                                                               random_state=rs)
    save('ar1_draws', **out)

    rej = {}
    for tag, a in (('test', TEST_AR1), ('q', QUANTILE)):
        m, res = rejection(a)
        rej.update({tag + '_observed': np.asarray(m.observed['AR1']), tag + '_n_sim': res.n_sim,
                    tag + '_threshold': res.threshold, tag + '_d': res.discrepancies,
                    tag + '_phi': np.asarray(res.samples['phi'])})
    save('ar1_rejection', **rej)

    c = COMPARE
    m = gauss.get_model(seed_obs=c['seed_obs'])
    res1 = elfi.Rejection(m['d'], seed=c['seeds'][0]).sample(c['n'])
    m['mu'].become(elfi.Prior('uniform', -10, 50))
    res2 = elfi.Rejection(m['d'], seed=c['seeds'][1]).sample(c['n'])
    m['gauss'].become(elfi.Simulator(ma2.MA2, m['mu'], m['sigma'], observed=m.observed['gauss']))
    res3 = elfi.Rejection(m['d'], seed=c['seeds'][2]).sample(c['n'])
    res = [res1, res2, res3]
    cmp = dict(p=elfi.compare_models(res), p_priors=elfi.compare_models(res, MODEL_PRIORS),
               model_priors=MODEL_PRIORS)
    for i, r in enumerate(res):
        cmp.update({'d{}'.format(i): r.discrepancies, 'n_samples{}'.format(i): r.n_samples,
                    'n_sim{}'.format(i): r.n_sim})
    save('compare_models', **cmp)


if __name__ == '__main__':
    main()
