"""Golden fixtures for the day care example, from the UNMODIFIED reference (elfi-dev/elfi, the
checkout named by ELFI_REFERENCE_ROOT).

    ELFI_REFERENCE_ROOT=<checkout> python tests/golden/gen_golden_daycare.py

* daycare_draws.npz     -- elfi.examples.daycare.daycare for seeded RandomStates: the default size
                           at the truth (batch 1 and 2), and a reduced size (5 DCCs of 12 children,
                           6 strains, a non-default freq_strains_commun, time_end 2) for a mixed
                           batch whose rows need very different numbers of transitions (the batch
                           lock-step matters) with the box corners t1, t2 or t3 = 0 and (11, 2, 1).
* daycare_summaries.npz -- the reference's four summaries of those draws and of crafted inputs
                           (all-zero data, one carrier of every strain, everyone carrying all).
* daycare_distance.npz  -- the reference's distance for B = 1 and B > 1, with an observed summary
                           whose maximum is 0, and NaN summaries.
* daycare_rejection.npz -- Rejection(daycare.get_model(seed_obs=..., time_end=0.05)['d'], ...)
                           .sample(...), as in the reference's test_daycare.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

from ref_shim import import_reference  # noqa: E402

elfi = import_reference()
from elfi.examples import daycare as dc  # noqa: E402

TRUTH = [3.6, 0.6, 0.1]
SMALL = dict(n_dcc=5, n_ind=12, n_strains=6, n_obs=9, time_end=2.0,
             freq_strains_commun=np.array([0.05, 0.1, 0.2, 0.02, 0.3, 0.15]))
MIXED = np.array([[3.6, 0.6, 0.1], [0.0, 0.6, 0.1], [3.6, 0.0, 0.1], [3.6, 0.6, 0.0],
                  [11.0, 2.0, 1.0], [0.5, 0.05, 0.9]])
REJECTION = dict(seed_obs=7, time_end=0.05, batch_size=10, seed=3, n=10, quantile=0.5)


def save(name, **arrays):
    np.savez_compressed(os.path.join(HERE, name + '.npz'), **arrays)
    print('wrote', name, {k: np.shape(v) for k, v in arrays.items()})


def summaries(x):
    return [dc.ss_shannon(x), dc.ss_strains(x), dc.ss_prevalence(x), dc.ss_prevalence_multi(x)]


def main():
    out = {}
    out['truth1'] = dc.daycare(*TRUTH, random_state=np.random.RandomState(1))
    out['truth2'] = dc.daycare(*TRUTH, batch_size=2, random_state=np.random.RandomState(2))
    out['mixed_prm'] = MIXED
    out['mixed'] = dc.daycare(*MIXED.T, batch_size=len(MIXED),
                              random_state=np.random.RandomState(3), **SMALL)
    out['small1'] = dc.daycare(*MIXED[4], random_state=np.random.RandomState(4), **SMALL)
    save('daycare_draws', **out)

    s = {}
    for name in ('truth1', 'truth2', 'mixed', 'small1'):
        s[name] = np.stack(summaries(out[name]))
    crafted = {'zeros': np.zeros((2, 3, 4, 5), dtype=bool),
               'diag': np.tile(np.eye(5, dtype=bool)[None, None], (1, 2, 1, 1)),
               'ones': np.ones((1, 4, 7, 9), dtype=bool)}
    crafted['diag'][0, 1, 0] = True
    for name, x in crafted.items():
        s['x_' + name] = x
        s[name] = np.stack(summaries(x))
    save('daycare_summaries', **s)

    d = {}
    obs = summaries(out['truth1'])
    sim = summaries(out['truth2'])
    d['d_truth_b2'] = dc.distance(*sim, observed=obs)
    d['d_truth_b1'] = dc.distance(*[v[:1] for v in sim], observed=obs)
    d['d_truth_b1_row1'] = dc.distance(*[v[1:] for v in sim], observed=obs)
    obs_small = summaries(out['small1'])
    sim_small = summaries(out['mixed'])
    obs_zero = [np.zeros_like(obs_small[0])] + obs_small[1:]
    d['obs_small'] = np.stack(obs_small)
    d['sim_small'] = np.stack(sim_small)
    d['d_small'] = dc.distance(*sim_small, observed=obs_small)
    d['d_small_obs0'] = dc.distance(*sim_small, observed=obs_zero)
    nan_sim = [v.astype(np.float64).copy() for v in sim_small]
    nan_sim[2][1, 3] = np.nan
    d['sim_nan'] = np.stack(nan_sim)
    d['d_nan'] = dc.distance(*nan_sim, observed=obs_small)
    save('daycare_distance', **d)

    r = REJECTION
    m = dc.get_model(seed_obs=r['seed_obs'], time_end=r['time_end'])
    res = elfi.Rejection(m['d'], batch_size=r['batch_size'], seed=r['seed']).sample(
        r['n'], quantile=r['quantile'])
    res_out = dict(n_sim=res.n_sim, threshold=res.threshold, d=res.discrepancies,
                   observed=np.asarray(m.observed['DCC']))
    for k, v in res.samples.items():
        res_out['out_' + k] = np.asarray(v)
    save('daycare_rejection', **res_out)


if __name__ == '__main__':
    main()
