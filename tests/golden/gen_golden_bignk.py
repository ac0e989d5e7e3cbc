"""Golden fixtures for the g-and-k summaries and the bivariate g-and-k example, from the UNMODIFIED
reference (elfi-dev/elfi, the checkout named by ELFI_REFERENCE_ROOT).

    ELFI_REFERENCE_ROOT=<checkout> python tests/golden/gen_golden_bignk.py

* bignk_draws.npz     -- elfi.examples.bignk.BiGNK for a seeded RandomState (per-row parameters,
                         including rho = 0 and rho near +-1) and gnk.GNK draws.
* bignk_summaries.npz -- gnk.ss_robust, gnk.ss_octile and gnk.euclidean_multiss of those draws
                         (d = 1 and d = 2) and of edge rows (ties, constant rows, +-inf, NaN).
* bignk_rejection.npz -- Rejection(bignk.get_model(seed=11)['d'], batch_size=10, seed=5).sample(20).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

from ref_shim import import_reference  # noqa: E402

elfi = import_reference()
from elfi.examples import bignk, gnk  # noqa: E402


def save(name, **arrays):
    np.savez(os.path.join(HERE, name + '.npz'), **arrays)
    print('wrote', name, {k: np.shape(v) for k, v in arrays.items()})


def edge_rows(n):
    """(6, n, 1) rows: ties, a constant row (ss_B = 0), +inf and -inf at every position, NaN."""
    rs = np.random.RandomState(n)
    rows = [np.round(rs.randn(n) * 2) / 2, np.full(n, 1.5), rs.randn(n), rs.randn(n),
            rs.randn(n), rs.randn(n)]
    rows[2][::3] = np.inf
    rows[3][1::2] = -np.inf
    rows[4][-1] = np.inf
    rows[5][n // 2] = np.nan
    return np.stack(rows)[:, :, None]


def main():
    prm = np.array([[3, 4, 1, 0.5, 1, 2, .5, .4, 0.6],
                    [0.5, 2, 3, 0.1, -2, 4, 0, 1.5, 0.0],
                    [4, 1, 0.2, 4, 3, -4, 2, -0.3, -0.99],
                    [1, 1, 1, 1, 0, 0, 0, 0, 0.999]]).T
    Yb = bignk.BiGNK(*prm, n_obs=40, batch_size=4, random_state=np.random.RandomState(3))
    gp = np.array([[3, 1, 2, .5], [1, 4, -1, 2], [0, 0.5, 0, 0]]).T
    Yg = gnk.GNK(*gp, n_obs=33, batch_size=3, random_state=np.random.RandomState(4))
    save('bignk_draws', prm=prm, bignk_y=Yb, gnk_prm=gp, gnk_y=Yg)

    out = {}
    for name, y in (('bignk', Yb), ('gnk', Yg), ('edge7', edge_rows(7)), ('edge50', edge_rows(50)),
                    ('edge1', edge_rows(1)), ('edge2', edge_rows(2))):
        with np.errstate(invalid='ignore'):
            r, o = gnk.ss_robust(y), gnk.ss_octile(y)
        out[name + '_y'] = y
        out[name + '_robust'] = r
        out[name + '_octile'] = o
        out[name + '_d_robust'] = gnk.euclidean_multiss(r, observed=[r[:1]])
        out[name + '_d_octile'] = gnk.euclidean_multiss(o, observed=[o[-1:]])
    save('bignk_summaries', **out)

    m = bignk.get_model(seed=11)
    res = elfi.Rejection(m['d'], batch_size=10, seed=5).sample(20)
    arrs = {'out_' + k: np.asarray(v) for k, v in res.samples.items()}
    save('bignk_rejection', n_sim=res.n_sim, threshold=res.threshold, out_d=res.discrepancies,
         observed_BiGNK=np.asarray(m.observed['BiGNK']), **arrs)


if __name__ == '__main__':
    main()
