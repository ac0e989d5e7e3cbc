"""Golden fixtures for the scratch assay example, from the UNMODIFIED reference (elfi-dev/elfi, the
checkout named by ELFI_REFERENCE_ROOT).

    ELFI_REFERENCE_ROOT=<checkout> python tests/golden/gen_golden_scratch_assay.py

* scratch_assay_draws.npz      -- the observed data of get_model(seed_obs=4) at the default size;
                                  cell_sim from a given init_arr; a batch of 8 through the
                                  vectorised simulator over the truth (0.25, 0.002), the prior
                                  corners (pm, pp in {0, 1}) and random parameters; a row whose
                                  lattice fills up (pp = 1); an empty initial lattice; a random
                                  reduced lattice (init_params=[8, 10, 20, 3]).
* scratch_assay_summaries.npz  -- cell_summaries of those draws and of crafted arrays.
* scratch_assay_rejection.npz  -- Rejection(get_model(init_params=[8, 10, 20, 3], seed_obs=1)['d'],
                                  batch_size=20, seed=3).sample(10, quantile=0.25), and that model's
                                  observed data and weights.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

from ref_shim import import_reference  # noqa: E402

elfi = import_reference()
from elfi.examples import scratch_assay as sa  # noqa: E402

TRUTH = (0.25, 0.002)
REDUCED = [8, 10, 20, 3]
BATCH = [TRUTH, (0.0, 0.0), (0.0, 1.0), (1.0, 0.0), (1.0, 1.0)]
REJECTION = dict(init_params=REDUCED, seed_obs=1, batch_size=20, seed=3, n=10, quantile=0.25)


def save(name, **arrays):
    np.savez_compressed(os.path.join(HERE, name + '.npz'), **arrays)
    print('wrote', name, {k: np.shape(v) for k, v in arrays.items()})


def crafted():
    rs = np.random.RandomState(11)
    x = (rs.uniform(size=(3, 4, 5, 6)) < 0.5).astype(np.float64)
    x[1] = 1.0                                  # constant frames: zero mismatches
    x[2, :, :, 1::2] = 1 - x[2, :, :, ::2]      # every site flips
    y = rs.uniform(-2, 2, size=(2, 3, 3, 4))    # not a lattice: the arithmetic itself
    return x, y


def main():
    m = sa.get_model(seed_obs=4)
    obs = np.asarray(m.observed['sim'])
    init = obs[0, :, :, 0]

    g = sa.cell_sim(*TRUTH, init_arr=init, random_state=np.random.RandomState(5))
    rs = np.random.RandomState(0)
    prm = np.array(BATCH + [tuple(rs.uniform(0, 1, 2)) for _ in range(3)])
    vec = elfi.tools.vectorize(sa.cell_sim, constants=(2,))
    batch = vec(prm[:, 0], prm[:, 1], init, random_state=np.random.RandomState(6))
    fill = sa.cell_sim(0.3, 1.0, init_arr=init, random_state=np.random.RandomState(7))
    empty = sa.cell_sim(0.5, 0.5, init_arr=np.zeros((6, 7)), random_state=np.random.RandomState(8))
    reduced = sa.cell_sim(0.4, 0.05, init_params=REDUCED, random_state=np.random.RandomState(9))
    save('scratch_assay_draws', obs=obs, given=g, prm=prm, batch=batch, fill=fill, empty=empty,
         reduced=reduced)

    x, y = crafted()
    out = dict(crafted=x, real=y)
    for name, arr in (('obs', obs), ('given', g[None]), ('batch', batch), ('fill', fill[None]),
                      ('empty', empty[None]), ('reduced', reduced[None]), ('crafted', x),
                      ('real', y)):
        out[name + '_sums'] = sa.cell_summaries(arr)
    save('scratch_assay_summaries', **out)

    a = REJECTION
    m = sa.get_model(init_params=a['init_params'], seed_obs=a['seed_obs'])
    res = elfi.Rejection(m['d'], batch_size=a['batch_size'], seed=a['seed']).sample(
        a['n'], quantile=a['quantile'])
    names = sorted(n for n in m.nodes if not n.startswith('_'))
    weights = m['d'].state['attr_dict']['_operation'].args[0].keywords['w']
    rej = dict(n_sim=res.n_sim, threshold=res.threshold, d=res.discrepancies,
               observed=np.asarray(m.observed['sim']), weights=np.asarray(weights),
               names=np.array(names))
    for k, v in res.samples.items():
        rej['out_' + k] = np.asarray(v)
    save('scratch_assay_rejection', **rej)


if __name__ == '__main__':
    main()
