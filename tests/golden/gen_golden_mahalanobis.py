"""Golden fixtures for Distance('mahalanobis', VI=...) on MA2, from the UNMODIFIED reference
(elfi-dev/elfi, the checkout named by ELFI_REFERENCE_ROOT).

    ELFI_REFERENCE_ROOT=<checkout> python tests/golden/gen_golden_mahalanobis.py

* ma2_mahalanobis.npz -- ma2.get_model(seed_obs=4) with its distance node replaced by
  Distance('mahalanobis', S1, S2, VI=VI).  VI is the inverse of the covariance of a prior-predictive
  pilot of (S1, S2): generate(PILOT_N, seed=PILOT_SEED), stored as `VI` next to the pilot's
  summaries.  Runs, each stored as <run>_t1, <run>_t2 (samples), <run>_d (discrepancies),
  <run>_n_sim and <run>_threshold:
    quantile   Rejection(batch_size=1000, seed=123).sample(100, quantile=0.01)
    nsim       Rejection(batch_size=500, seed=7).sample(64, n_sim=3000)
    threshold  Rejection(batch_size=1000, seed=123).sample(150, threshold=0.3)
    smc        SMC(batch_size=1000, seed=20).sample(150, thresholds=[1.0, 0.5]), with the final
               weights as smc_weights and per population pop<i>_t1, pop<i>_t2, pop<i>_d,
               pop<i>_weights, pop<i>_n_sim, pop<i>_threshold.
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

PILOT_N = 2000
PILOT_SEED = 99
REJECTION = {'quantile': (dict(batch_size=1000, seed=123), dict(n_samples=100, quantile=0.01)),
             'nsim': (dict(batch_size=500, seed=7), dict(n_samples=64, n_sim=3000)),
             'threshold': (dict(batch_size=1000, seed=123), dict(n_samples=150, threshold=0.3))}
SMC = (dict(batch_size=1000, seed=20), dict(n_samples=150, thresholds=[1.0, 0.5]))


def model(VI=None):
    """MA2 (seed_obs=4) with d = Distance('mahalanobis', S1, S2, VI=VI); with VI None, the pilot's
    VI and summaries as well."""
    m = ma2.get_model(seed_obs=4)
    pilot = None
    if VI is None:
        out = m.generate(PILOT_N, ['S1', 'S2'], seed=PILOT_SEED)
        pilot = np.column_stack([np.asarray(out['S1']).ravel(), np.asarray(out['S2']).ravel()])
        VI = np.linalg.inv(np.cov(pilot, rowvar=False))
    m['d'].become(elfi.Distance('mahalanobis', m['S1'], m['S2'], VI=VI))
    return m, VI, pilot


def run_arrays(prefix, res):
    return {prefix + 't1': np.asarray(res.samples['t1']), prefix + 't2': np.asarray(res.samples['t2']),
            prefix + 'd': np.asarray(res.discrepancies), prefix + 'n_sim': np.int64(res.n_sim),
            prefix + 'threshold': np.float64(res.threshold)}


def main():
    m, VI, pilot = model()
    out = dict(VI=VI, pilot=pilot, pilot_n=np.int64(PILOT_N), pilot_seed=np.int64(PILOT_SEED))
    for name, (init, kw) in REJECTION.items():
        res = elfi.Rejection(m['d'], **init).sample(bar=False, **kw)
        out.update(run_arrays(name + '_', res))
    res = elfi.SMC(m['d'], **SMC[0]).sample(bar=False, **SMC[1])
    out.update(run_arrays('smc_', res))
    out['smc_weights'] = np.asarray(res.weights)
    out['smc_n_pops'] = np.int64(len(res.populations))
    for i, pop in enumerate(res.populations):
        out.update(run_arrays('pop{}_'.format(i), pop))
        out['pop{}_weights'.format(i)] = np.asarray(pop.weights)
    np.savez(os.path.join(HERE, 'ma2_mahalanobis.npz'), **out)
    print('wrote ma2_mahalanobis', {k: np.shape(v) for k, v in out.items()})


if __name__ == '__main__':
    main()
