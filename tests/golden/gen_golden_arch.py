"""Golden fixtures for the ARCH(1) example, from the UNMODIFIED reference (elfi-dev/elfi, the checkout
named by ELFI_REFERENCE_ROOT).

    ELFI_REFERENCE_ROOT=<checkout> python tests/golden/gen_golden_arch.py

* arch_draws.npz     -- elfi.examples.arch.arch for seeded RandomStates: one row at the truth
                        (0.3, 0.7); a batch over the truth, the corners t1 = +-1, t2 in {0, 1} and
                        random parameters; the same batch at n_obs = 17.
* arch_summaries.npz -- sample_mean, sample_variance, autocorr and pairwise_autocorr (as the
                        (B, 2 + L + L(L-1)/2) matrix of get_model's order) of those draws with L = 5
                        and 8, and of crafted rows: constant, zero, with NaN, with +-inf, n = 2
                        (L = 1) and n = 128 (L = 8).
* arch_rejection.npz -- Rejection(arch.get_model(seed_obs=...)['d'], ...).sample(...), and the
                        n_obs quirk: get_model(n_obs=40)'s observed series and a generated batch of
                        its simulator and distance.
"""
import os
import sys
from itertools import combinations

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

from ref_shim import import_reference  # noqa: E402

elfi = import_reference()
from elfi.examples import arch  # noqa: E402

TRUTH = (0.3, 0.7)
CORNERS = [(1., 0.), (1., 1.), (-1., 0.), (-1., 1.)]
REJECTION = dict(seed_obs=1, batch_size=100, seed=3, n=20, quantile=0.1)
QUIRK = dict(n_obs=40, seed_obs=2, batch_size=4, seed=5)


def save(name, **arrays):
    np.savez(os.path.join(HERE, name + '.npz'), **arrays)
    print('wrote', name, {k: np.shape(v) for k, v in arrays.items()})


def summaries(x, n_lags):
    """The summaries of get_model's graph, in its order, as columns."""
    cols = [arch.sample_mean(x), arch.sample_variance(x)]
    cols += [arch.autocorr(x, i) for i in range(1, n_lags + 1)]
    cols += [arch.pairwise_autocorr(x, i, j) for i, j in combinations(range(1, n_lags + 1), 2)]
    return np.column_stack(cols)


def crafted():
    rs = np.random.RandomState(11)
    x = rs.randn(8, 100)
    x[0] = 2.5                       # constant: std 0, AC and PW are NaN
    x[1] = 0.0                       # zero row: mean 0, NaN correlations
    x[2, 17] = np.nan
    x[3, 50] = np.inf
    x[4, 3] = -np.inf
    x[5] = x[5] * 1e150              # squares overflow to inf
    x[6] = -x[6] * 1e-160            # squares underflow: tiny and zero terms
    x[7, :50] = -0.0                 # signed zeros next to values
    x[7, 50:] = 0.0
    return x


def main():
    y1 = arch.arch(*TRUTH, batch_size=1, random_state=np.random.RandomState(1))
    rs = np.random.RandomState(0)
    prm = np.array([TRUTH] + CORNERS + list(zip(rs.uniform(-1, 1, 11), rs.uniform(0, 1, 11))))
    yb = arch.arch(prm[:, 0], prm[:, 1], batch_size=len(prm), random_state=np.random.RandomState(2))
    ys = arch.arch(prm[:, 0], prm[:, 1], n_obs=17, batch_size=len(prm),
                   random_state=np.random.RandomState(3))
    save('arch_draws', y1=y1, prm=prm, yb=yb, ys=ys)

    rs = np.random.RandomState(5)
    n2 = rs.randn(6, 2)
    n2[0] = 1.0
    n2[1, 1] = np.nan
    n128 = rs.randn(6, 128) * rs.uniform(0.1, 10, (6, 1))
    n128[0] = -3.0
    n128[1, 127] = np.inf
    out = dict(crafted=crafted(), n2=n2, n128=n128)
    with np.errstate(all='ignore'):
        for name, x, lags in (('y1', y1, (5, 8)), ('yb', yb, (5, 8)), ('ys', ys, (5, 8)),
                              ('crafted', out['crafted'], (5, 8)), ('n2', n2, (1,)),
                              ('n128', n128, (1, 8))):
            for L in lags:
                out['{}_L{}'.format(name, L)] = summaries(x, L)
    save('arch_summaries', **out)

    a = REJECTION
    m = arch.get_model(seed_obs=a['seed_obs'])
    res = elfi.Rejection(m['d'], batch_size=a['batch_size'], seed=a['seed']).sample(
        a['n'], quantile=a['quantile'])
    rej = dict(n_sim=res.n_sim, threshold=res.threshold, d=res.discrepancies,
               observed=np.asarray(m.observed['Y']))
    for k, v in res.samples.items():
        rej['out_' + k] = np.asarray(v)
    q = QUIRK
    mq = arch.get_model(n_obs=q['n_obs'], seed_obs=q['seed_obs'])
    gen = mq.generate(q['batch_size'], outputs=['t1', 't2', 'Y', 'd'], seed=q['seed'])
    rej.update(quirk_observed=np.asarray(mq.observed['Y']), quirk_t1=gen['t1'], quirk_t2=gen['t2'],
               quirk_Y=gen['Y'], quirk_d=gen['d'])
    save('arch_rejection', **rej)


if __name__ == '__main__':
    main()
