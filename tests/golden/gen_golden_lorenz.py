"""Golden fixtures for the Lorenz example, from the UNMODIFIED reference (elfi-dev/elfi, the checkout
named by ELFI_REFERENCE_ROOT).

    ELFI_REFERENCE_ROOT=<checkout> python tests/golden/gen_golden_lorenz.py

* lorenz_draws.npz     -- elfi.examples.lorenz.forecast_lorenz for a seeded RandomState over a
                          parameter grid with the prior's four corners and the true parameters, at
                          n_timestep = 16 and total_duration = 0.4 (the default step of 0.025; at
                          the default duration a step of 0.25 overflows to NaN within 4 steps); at
                          phi = 1.5 (NaN rows); and two noise-free rows
                          (phi = 1, so eta stays exactly 0) at the default length of 160 steps.
* lorenz_summaries.npz -- the reference's mean, var, autocov, cov, xcov(prev=True / False) of those
                          draws and of crafted inputs: rows with a NaN, with +inf, with -inf and +inf,
                          constant rows, and T = 2 rows, for n_obs in {4, 7, 40}.
* lorenz_rejection.npz -- Rejection(lorenz.get_model(seed_obs=...)['d'], ...).sample(...).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

from ref_shim import import_reference  # noqa: E402

elfi = import_reference()
from elfi.examples import lorenz  # noqa: E402

# (theta1, theta2): the prior's corners, the truth, two inner points
PRM = np.array([[0.5, 0.0], [0.5, 0.3], [3.5, 0.0], [3.5, 0.3], [2.0, 0.1], [1.2, 0.25]])
NOISE_FREE_PRM = np.array([[2.0, 0.1], [0.7, 0.28]])
REJECTION = dict(seed_obs=7, batch_size=10, seed=3, n=10)


def save(name, **arrays):
    np.savez_compressed(os.path.join(HERE, name + '.npz'), **arrays)
    print('wrote', name, {k: np.shape(v) for k, v in arrays.items()})


def summaries(x):
    with np.errstate(invalid='ignore', over='ignore'):
        return np.column_stack([lorenz.mean(x), lorenz.var(x), lorenz.autocov(x), lorenz.cov(x),
                                lorenz.xcov(x, True), lorenz.xcov(x, False)])


def crafted():
    """(name, x) inputs of the summaries that the simulator does not produce."""
    rs = np.random.RandomState(5)
    out = []
    for m in (4, 7, 40):
        x = rs.randn(6, 9, m) * 3.0
        x[0, 4, 1] = np.nan
        x[1, 0, 2] = np.inf
        x[2, 3, 0], x[2, 5, 3] = -np.inf, np.inf
        x[3] = 2.5
        x[4] = -0.0
        x[5, :, 1] = 1e300
        out.append(('m{}'.format(m), x))
        out.append(('t2_m{}'.format(m), rs.randn(3, 2, m)))
    return out


def main():
    rs = np.random.RandomState(3)
    x = lorenz.forecast_lorenz(*PRM.T, n_timestep=16, total_duration=0.4, batch_size=len(PRM),
                               random_state=rs)
    with np.errstate(invalid='ignore'):
        xnan = lorenz.forecast_lorenz(2.0, 0.1, phi=1.5, n_timestep=4, batch_size=2,
                                      random_state=np.random.RandomState(4))
    xfree = lorenz.forecast_lorenz(*NOISE_FREE_PRM.T, phi=1.0, batch_size=len(NOISE_FREE_PRM),
                                   random_state=np.random.RandomState(5))
    save('lorenz_draws', prm=PRM, x=x, x_phi15=xnan, noise_free_prm=NOISE_FREE_PRM,
         x_noise_free=xfree)

    out = {'draws': summaries(x), 'noise_free': summaries(xfree)}
    for name, c in crafted():
        out['x_' + name] = c
        out['s_' + name] = summaries(c)
    save('lorenz_summaries', **out)

    a = REJECTION
    m = lorenz.get_model(seed_obs=a['seed_obs'])
    res = elfi.Rejection(m['d'], batch_size=a['batch_size'], seed=a['seed']).sample(a['n'])
    res_out = dict(n_sim=res.n_sim, threshold=res.threshold, d=res.discrepancies,
                   observed=np.asarray(m.observed['Lorenz']))
    for k, v in res.samples.items():
        res_out['out_' + k] = np.asarray(v)
    save('lorenz_rejection', **res_out)


if __name__ == '__main__':
    main()
