"""Golden fixtures for the M/G/1 example, from the UNMODIFIED reference (elfi-dev/elfi, the checkout
named by ELFI_REFERENCE_ROOT).

    ELFI_REFERENCE_ROOT=<checkout> python tests/golden/gen_golden_mg1.py

* mg1_draws.npz        -- elfi.examples.mg1.MG1 for seeded RandomStates: one row at the truth
                          (1, 5, 0.2); a batch of 16 over the truth, the prior corners (t3 near 0
                          and at 0.5, t2 = t1, t2 = t1 + 10) and random parameters; the same batch
                          at n_obs = 7.
* mg1_summaries.npz    -- log_identity and quantiles (10 levels) of those draws, and quantiles of
                          crafted rows: ties, NaN, +-inf, n = 2, with 10 and with random levels.
* mg1_prior_logpdf.npz -- the reference ModelPrior(get_model()).logpdf at points inside the support,
                          on each edge, one ulp beyond, and with t2 < t1.
* mg1_rejection.npz    -- Rejection(mg1.get_model(seed_obs=...)['d'], ...).sample(..., quantile=...).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

from ref_shim import import_reference  # noqa: E402

elfi = import_reference()
from elfi.examples import mg1  # noqa: E402
from elfi.model.extensions import ModelPrior  # noqa: E402

TRUTH = (1., 5., 0.2)
CORNERS = [(1., 5., 1e-3), (1., 5., 0.5), (3., 3., 0.2), (3., 13., 0.2), (0., 0., 1e-3),
           (10., 20., 0.5)]
REJECTION = dict(seed_obs=1, batch_size=100, seed=3, n=20, quantile=0.1)


def save(name, **arrays):
    np.savez(os.path.join(HERE, name + '.npz'), **arrays)
    print('wrote', name, {k: np.shape(v) for k, v in arrays.items()})


def crafted():
    rs = np.random.RandomState(11)
    x = rs.exponential(2.0, (10, 50))
    x[0] = 2.5                       # constant
    x[1, ::2] = x[1, 1::2]           # ties in pairs
    x[2, 17] = np.nan
    x[3, 20] = np.inf
    x[4, 3] = -np.inf
    x[5, :3] = [np.inf, -np.inf, 1.0]  # inf - inf at the interpolation
    x[6] = np.round(x[6])            # many ties
    x[7, :25] = -0.0
    x[7, 25:] = 0.0
    x[8, 5] = np.nan
    x[8, 6] = np.inf
    return x


def main():
    y1 = mg1.MG1(*TRUTH, batch_size=1, random_state=np.random.RandomState(1))
    rs = np.random.RandomState(0)
    t1 = rs.uniform(0, 10, 9)
    rand = np.column_stack([t1, t1 + rs.uniform(0, 10, 9), rs.uniform(0, 0.5, 9)])
    prm = np.array([TRUTH] + CORNERS + list(rand))
    yb = mg1.MG1(prm[:, 0], prm[:, 1], prm[:, 2], batch_size=len(prm),
                 random_state=np.random.RandomState(2))
    ys = mg1.MG1(prm[:, 0], prm[:, 1], prm[:, 2], n_obs=7, batch_size=len(prm),
                 random_state=np.random.RandomState(3))
    save('mg1_draws', y1=y1, prm=prm, yb=yb, ys=ys)

    q10 = np.linspace(0, 1, 10)
    rs = np.random.RandomState(5)
    qr = np.sort(rs.uniform(0, 1, 7))
    n2 = rs.exponential(1.0, (6, 2))
    n2[0] = 1.0
    n2[1, 1] = np.nan
    n2[2] = [np.inf, 1.0]
    out = dict(crafted=crafted(), n2=n2, qr=qr)
    with np.errstate(all='ignore'):
        for name, x in (('y1', y1), ('yb', yb), ('ys', ys)):
            out[name + '_log'] = mg1.log_identity(x)
            out[name + '_q10'] = mg1.quantiles(x, q10)
        for name in ('crafted', 'n2'):
            out[name + '_q10'] = mg1.quantiles(out[name], q10)
            out[name + '_qr'] = mg1.quantiles(out[name], qr)
    save('mg1_summaries', **out)

    m = mg1.get_model(seed_obs=1)
    up = np.nextafter
    pts = [[1., 5., 0.2], [0., 0., 0.], [10., 20., 0.5], [0., 10., 0.5], [10., 10., 0.],
           [2., 2., 0.1], [2., 12., 0.1], [2., up(12., 13.), 0.1], [2., up(2., 1.), 0.1],
           [up(0., -1.), 5., 0.1], [up(10., 11.), 15., 0.1], [3., 4., up(0.5, 1.)],
           [3., 4., up(0., -1.)], [5., 4., 0.2], [5., 1., 0.2], [-1., 0.5, 0.2]]
    rs = np.random.RandomState(7)
    t1 = rs.uniform(-1, 11, 40)
    pts += list(np.column_stack([t1, t1 + rs.uniform(-2, 12, 40), rs.uniform(-0.1, 0.6, 40)]))
    x = np.array(pts)
    with np.errstate(all='ignore'):
        lp = ModelPrior(m).logpdf(x)
    save('mg1_prior_logpdf', x=x, logpdf=lp, names=np.array(m.parameter_names))

    a = REJECTION
    m = mg1.get_model(seed_obs=a['seed_obs'])
    res = elfi.Rejection(m['d'], batch_size=a['batch_size'], seed=a['seed']).sample(
        a['n'], quantile=a['quantile'])
    rej = dict(n_sim=res.n_sim, threshold=res.threshold, d=res.discrepancies,
               observed=np.asarray(m.observed['MG1']))
    for k, v in res.samples.items():
        rej['out_' + k] = np.asarray(v)
    save('mg1_rejection', **rej)


if __name__ == '__main__':
    main()
