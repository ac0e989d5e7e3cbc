"""Golden fixtures for the birth-death-mutation example, from the UNMODIFIED reference (elfi-dev/elfi,
the checkout named by ELFI_REFERENCE_ROOT) and its C++ simulator as oracle/ref_bins.mk builds it
(oracle/_ref/bdm, from elfi/examples/cpp/bdm.cpp).

    ELFI_REFERENCE_ROOT=<checkout> make -C oracle -f ref_bins.mk
    ELFI_REFERENCE_ROOT=<checkout> python tests/golden/gen_golden_bdm.py

The reference's model runs in a temporary working directory that holds a copy of the executable.

* bdm_draws.npz     -- get_model().generate(B, ['BDM', 'T1', 'd'], seed=s) for a few (B, s).
* bdm_summaries.npz -- the reference's T1 and T2 on crafted int16 matrices: an extinct row, N = 1,
                       N = 473, and T2 with n != 20.
* bdm_rejection.npz -- Rejection(get_model()['d'], batch_size=1000, seed=1).sample(200,
                       quantile=0.1): samples, threshold, discrepancies.
* bdm_law.npz       -- 2e4 executable rows (one seed) at each of four parameter points with four
                       decimals; per row only T1, the number of clusters and the population.
"""
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

from ref_shim import import_reference  # noqa: E402

elfi = import_reference()
from elfi.examples import bdm  # noqa: E402

EXE = os.path.join(ROOT, 'oracle', '_ref', 'bdm')
DRAWS = ((1, 1), (7, 2), (300, 3))
REJECTION = dict(batch_size=1000, seed=1, n=200, quantile=0.1)
# (alpha, delta, tau, N): the example's truth, a birth-poor point, extinctions, Tanaka's N
LAW_POINTS = np.array([[0.2, 0.0, 0.198, 20], [0.005, 0.0, 0.198, 20], [1.0, 0.3, 0.198, 20],
                       [1.0, 0.1, 0.198, 473]])
LAW_ROWS = 20000
LAW_SEEDS = (11, 12, 13, 14)


def save(name, **arrays):
    np.savez_compressed(os.path.join(HERE, name + '.npz'), **arrays)
    print('wrote', name, {k: np.shape(v) for k, v in arrays.items()})


def law_rows(point, seed, workdir):
    """LAW_ROWS executable rows at one point: (T1, clusters, pop) per row."""
    inp = os.path.join(workdir, 'law.txt')
    np.savetxt(inp, np.tile(point, (LAW_ROWS, 1)), fmt='%.4f %.4f %.4f %d')
    out = subprocess.run([EXE, inp, '--seed', str(seed), '--mode', '1'], check=True,
                         stdout=subprocess.PIPE).stdout
    c = np.loadtxt(out.decode().splitlines(), dtype=np.int64, ndmin=2)
    assert c.shape == (LAW_ROWS, int(point[3]))
    pop = c.sum(axis=1)
    clusters = (c > 0).sum(axis=1)
    with np.errstate(invalid='ignore'):
        t1 = clusters / pop
    return t1, clusters, pop


def main():
    if not os.path.isfile(EXE):
        raise SystemExit('build the executable first: ELFI_REFERENCE_ROOT=... make -C oracle -f '
                         'ref_bins.mk')
    cwd = os.getcwd()
    work = tempfile.mkdtemp()
    try:
        shutil.copy(EXE, os.path.join(work, 'bdm'))
        os.chdir(work)
        out = {}
        m = bdm.get_model()
        out['observed'] = np.asarray(m.observed['BDM'])
        for B, s in DRAWS:
            g = m.generate(B, ['BDM', 'T1', 'd'], seed=s)
            for k in ('BDM', 'T1', 'd'):
                out['{}_B{}_s{}'.format(k, B, s)] = np.asarray(g[k])
        save('bdm_draws', **out)

        r = REJECTION
        res = elfi.Rejection(m['d'], batch_size=r['batch_size'], seed=r['seed']).sample(
            r['n'], quantile=r['quantile'])
        save('bdm_rejection', alpha=np.asarray(res.samples['alpha']), threshold=res.threshold,
             d=res.discrepancies, n_sim=res.n_sim)

        law = {'points': LAW_POINTS, 'seeds': np.array(LAW_SEEDS)}
        for i, (point, seed) in enumerate(zip(LAW_POINTS, LAW_SEEDS)):
            law['t1_%d' % i], law['clusters_%d' % i], law['pop_%d' % i] = law_rows(point, seed,
                                                                                 work)
        save('bdm_law', **law)
    finally:
        os.chdir(cwd)
        shutil.rmtree(work)

    rs = np.random.RandomState(5)
    crafted = {
        'extinct': np.array([[0] * 20, [6, 3, 2, 2, 1, 1, 1, 1, 1, 1, 1] + [0] * 9,
                             [0, 0, 4, 0, 1] + [0] * 15], dtype=np.int16),
        'n1': np.array([[0], [1], [7]], dtype=np.int16),
        'n473': rs.randint(0, 4, (5, 473)).astype(np.int16),
        'n1024': rs.randint(0, 3, (3, 1024)).astype(np.int16),
        'n20': rs.randint(0, 6, (6, 20)).astype(np.int16),
    }
    s = {}
    with np.errstate(all='ignore'):
        for name, x in crafted.items():
            s['x_' + name] = x
            s['t1_' + name] = bdm.T1(x)
            s['t2_' + name] = bdm.T2(x)
            s['t2n7_' + name] = bdm.T2(x, n=7)
            s['t2n473_' + name] = bdm.T2(x, n=473)
    save('bdm_summaries', **s)


if __name__ == '__main__':
    main()
