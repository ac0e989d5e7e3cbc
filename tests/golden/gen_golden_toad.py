"""Golden fixtures for the toad example, from the UNMODIFIED reference (elfi-dev/elfi, the checkout
named by ELFI_REFERENCE_ROOT).

    ELFI_REFERENCE_ROOT=<checkout> python tests/golden/gen_golden_toad.py

* toad_draws.npz     -- elfi.examples.toad.toad for a seeded RandomState at 5 toads x 9 days over a
                        parameter grid with the prior's corners (alpha = 1 exactly, gamma = 0,
                        p0 = 0), the true parameters and inner points; a batch where every gamma is
                        0 (SciPy then returns zero steps without drawing, and alpha = 1 makes them
                        NaN); and the true parameters at the default 66 toads x 63 days.
* toad_summaries.npz -- the reference's compute_summaries of those draws for every lag, and of
                        crafted inputs: every toad returned, NaN and +-inf positions, 1.5e308 steps
                        with 594 and 605 displacement rows (both sides of nanmedian's switch at
                        600), and non-default p and thd.
* toad_rejection.npz -- Rejection(toad.get_model(seed_obs=...)['d'], ...).sample(...).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

from ref_shim import import_reference  # noqa: E402

elfi = import_reference()
from elfi.examples import toad  # noqa: E402

# (alpha, gamma, p0): the prior's corners, the truth, inner points
PRM = np.array([[1.0, 0.0, 0.0], [1.0, 0.0, 0.9], [1.0, 100.0, 0.0], [1.0, 100.0, 0.9],
                [2.0, 0.0, 0.0], [2.0, 0.0, 0.9], [2.0, 100.0, 0.0], [2.0, 100.0, 0.9],
                [1.7, 35.0, 0.6], [1.3, 5.0, 0.2], [1.0, 20.0, 0.5], [1.99, 60.0, 0.3]])
ZERO_GAMMA_PRM = np.array([[1.0, 0.0, 0.3], [1.5, 0.0, 0.3]])
SMALL = dict(n_toads=5, n_days=9)
REJECTION = dict(seed_obs=7, batch_size=10, seed=3, n=10)


def save(name, **arrays):
    np.savez_compressed(os.path.join(HERE, name + '.npz'), **arrays)
    print('wrote', name, {k: np.shape(v) for k, v in arrays.items()})


def crafted():
    """(name, x, lag, p, thd) inputs of the summaries that the simulator does not produce."""
    rs = np.random.RandomState(11)
    p = np.linspace(0, 1, 11)
    out = [('returned', np.zeros((9, 5, 3)), 1, p, 10)]
    x = np.cumsum(rs.standard_cauchy((9, 5, 6)) * 30, axis=0)
    x[3, 1, 0] = np.nan
    x[:, :, 1] = np.nan
    x[5, 2, 2] = np.inf
    x[2, 0, 3], x[6, 4, 3] = -np.inf, np.inf
    x[:, 1:, 4] = 0.0                    # one toad moves: few kept values
    x[:, :, 5] = 0.0
    x[4, 3, 5] = 50.0                    # a single kept value per lag
    for lag in (1, 2, 3, 8):
        out.append(('naninf_lag{}'.format(lag), x, lag, p, 10))
    for n_toads in (54, 55):             # 11 * n_toads = 594 and 605 displacement rows
        big = np.zeros((12, n_toads, 3))
        big[:, 0, 0] = 1.5e308 * (np.arange(12) % 2)          # 11 kept values, all 1.5e308
        big[:, 0, 1] = 1.5e308 * (np.arange(12) % 2)
        big[:, 1, 1] = 20.0 * (np.arange(12) % 3)              # 11 + 11 kept values
        big[:, :, 2] = np.cumsum(rs.standard_normal((12, n_toads)) * 40, axis=0)
        out.append(('big{}'.format(n_toads), big, 1, p, 10))
    y = np.cumsum(rs.standard_normal((9, 5, 4)) * 20, axis=0)
    out.append(('p_thd', y, 2, np.array([0.05, 0.5, 0.25, 0.95, 1.0]), 3.5))
    out.append(('p_one', y, 1, np.array([1.0]), 0.0))
    out.append(('p_thd_neg', y, 3, np.array([0.0, 0.3, 0.7]), -1.0))
    return out


def main():
    x = toad.toad(*PRM.T, batch_size=len(PRM), random_state=np.random.RandomState(3), **SMALL)
    with np.errstate(invalid='ignore'):
        xz = toad.toad(*ZERO_GAMMA_PRM.T, batch_size=len(ZERO_GAMMA_PRM),
                       random_state=np.random.RandomState(4), **SMALL)
    xt = toad.toad(1.7, 35.0, 0.6, batch_size=3, random_state=np.random.RandomState(5))
    save('toad_draws', prm=PRM, x=x, zero_gamma_prm=ZERO_GAMMA_PRM, x_zero_gamma=xz, x_true=xt)

    out = {}
    with np.errstate(invalid='ignore', over='ignore'):
        for lag in range(1, SMALL['n_days']):
            out['draws_lag{}'.format(lag)] = toad.compute_summaries(x, lag)
        for lag in (1, 2, 4, 8):
            out['true_lag{}'.format(lag)] = toad.compute_summaries(xt, lag)
        for name, c, lag, p, thd in crafted():
            out['x_' + name] = c
            out['lag_' + name] = np.int64(lag)
            out['p_' + name] = p
            out['thd_' + name] = np.float64(thd)
            out['s_' + name] = toad.compute_summaries(c, lag, p=p, thd=thd)
    save('toad_summaries', **out)

    a = REJECTION
    m = toad.get_model(seed_obs=a['seed_obs'])
    res = elfi.Rejection(m['d'], batch_size=a['batch_size'], seed=a['seed']).sample(a['n'])
    res_out = dict(n_sim=res.n_sim, threshold=res.threshold, d=res.discrepancies,
                   observed=np.asarray(m.observed['toad']))
    for k, v in res.samples.items():
        res_out['out_' + k] = np.asarray(v)
    save('toad_rejection', **res_out)


if __name__ == '__main__':
    main()
