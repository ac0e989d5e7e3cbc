"""Golden fixtures for the alpha-stable stochastic volatility example, from the UNMODIFIED reference
(elfi-dev/elfi, the checkout named by ELFI_REFERENCE_ROOT).

    ELFI_REFERENCE_ROOT=<checkout> python tests/golden/gen_golden_svm.py

* svm_draws.npz      -- alpha_stochastic_volatility_model for seeded RandomStates: one row at the
                        truth (1.2, 0.5); a batch of 24 over the truth, the prior corners (alpha at
                        0.5, 1.0 exactly and 2.0; beta at -1, 0, -0.0 and 1) and random parameters;
                        one call with x_0 given.
* svm_summaries.npz  -- kurt and skew of those draws, and of crafted rows: ties, NaN, +-inf,
                        q75 == q25 (division by zero), n = 2.
* svm_rejection.npz  -- Rejection(get_model(seed_obs=1)['d'], batch_size=100, seed=3)
                        .sample(20, quantile=0.1).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

from ref_shim import import_reference  # noqa: E402

elfi = import_reference()
from elfi.examples import stochastic_volatility_model as svm  # noqa: E402

TRUTH = (1.2, 0.5)
FIXED = dict(kappa=1, eta=0, mu=0, phi=0.95, sigma=0.2)
CORNERS = [(0.5, -1.0), (0.5, 0.0), (0.5, 1.0), (1.0, -1.0), (1.0, 0.0), (1.0, -0.0), (1.0, 1.0),
           (1.0, 0.5), (2.0, -1.0), (2.0, 0.0), (2.0, 1.0), (1.2, -0.0)]
REJECTION = dict(seed_obs=1, batch_size=100, seed=3, n=20, quantile=0.1)


def save(name, **arrays):
    np.savez(os.path.join(HERE, name + '.npz'), **arrays)
    print('wrote', name, {k: np.shape(v) for k, v in arrays.items()})


def crafted():
    rs = np.random.RandomState(11)
    x = rs.standard_cauchy((10, 50))
    x[0] = 2.5                       # constant: 0 / 0
    x[1, ::2] = x[1, 1::2]           # ties in pairs
    x[2, 17] = np.nan
    x[3, 20] = np.inf
    x[4, 3] = -np.inf
    x[5, :3] = [np.inf, -np.inf, 1.0]
    x[6] = np.round(x[6])            # many ties
    x[7, :45] = 1.0                  # q75 == q25 but not q95 == q05: division by zero
    x[8, 10:40] = 0.0                # q75 == q25 == 0
    x[9, :5] = -0.0
    return x


def main():
    y1 = svm.alpha_stochastic_volatility_model(*TRUTH, **FIXED, batch_size=1,
                                               random_state=np.random.RandomState(1))
    rs = np.random.RandomState(0)
    rand = np.column_stack([rs.uniform(0.5, 2.0, 11), rs.uniform(-1, 1, 11)])
    prm = np.array([TRUTH] + CORNERS + list(rand))
    yb = svm.alpha_stochastic_volatility_model(prm[:, 0], prm[:, 1], **FIXED, batch_size=len(prm),
                                               random_state=np.random.RandomState(2))
    yx = svm.alpha_stochastic_volatility_model(prm[:, 0], prm[:, 1], **FIXED, n_obs=20, x_0=0.3,
                                               batch_size=len(prm),
                                               random_state=np.random.RandomState(3))
    save('svm_draws', y1=y1, prm=prm, yb=yb, yx=yx)

    rs = np.random.RandomState(5)
    n2 = rs.standard_cauchy((4, 2))
    n2[0] = 1.0
    n2[1, 1] = np.nan
    out = dict(crafted=crafted(), n2=n2)
    with np.errstate(all='ignore'):
        for name, x in (('y1', y1), ('yb', yb), ('yx', yx)):
            out[name + '_kurt'] = svm.kurt(x)
            out[name + '_skew'] = svm.skew(x)
        for name in ('crafted', 'n2'):
            out[name + '_kurt'] = svm.kurt(out[name])
            out[name + '_skew'] = svm.skew(out[name])
    save('svm_summaries', **out)

    a = REJECTION
    m = svm.get_model(seed_obs=a['seed_obs'])
    res = elfi.Rejection(m['d'], batch_size=a['batch_size'], seed=a['seed']).sample(
        a['n'], quantile=a['quantile'])
    names = sorted(n for n in m.nodes if not n.startswith('_'))     # without the hidden nodes
    rej = dict(n_sim=res.n_sim, threshold=res.threshold, d=res.discrepancies,
               observed=np.asarray(m.observed['a_svm']), names=np.array(names))
    for k, v in res.samples.items():
        rej['out_' + k] = np.asarray(v)
    save('svm_rejection', **rej)


if __name__ == '__main__':
    main()
