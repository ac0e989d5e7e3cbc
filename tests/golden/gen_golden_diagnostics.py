"""Golden fixtures for TwoStageSelection, from the UNMODIFIED reference (elfi-dev/elfi, the checkout
named by ELFI_REFERENCE_ROOT).

    ELFI_REFERENCE_ROOT=<checkout> python tests/golden/gen_golden_diagnostics.py

diagnostics.npz holds three groups of cases.
* ma2_*    -- the reference's unit-test model (MA2 with ac_lag1, ac_lag2 and ss_mean, y_obs from
              RandomState(0)) at n_sim = 20000, batch_size = 2000, seed 0: per combination the
              accepted parameters (_obtain_accepted_thetas), _calc_entropy and _calc_MRSSE, and the
              index of the combination run() selects.
* twice_*  -- prepared_ss = [(ac_lag1,), (ac_lag1, ac_lag2), (ac_lag1,)] on the same model,
  round_*  -- candidates rounded to one decimal, so that distances tie,
  dup_*    -- priors randint(-1, 2) and randint(0, 2), so accepted parameters repeat (entropy
              -inf); each at n_sim = 5000, batch_size = 1000, seed 1, with the same records.
* pts_*    -- _calc_entropy and _calc_MRSSE on crafted point sets, q = 1 .. 6, k = 2, 4, 8, with
              duplicated points and sets of fewer than k points.
"""
import os
import sys
from functools import partial

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

from ref_shim import import_reference  # noqa: E402

elfi = import_reference()
import elfi.examples.gauss as Gauss  # noqa: E402
import elfi.examples.ma2 as MA2  # noqa: E402
from elfi.methods.diagnostics import TwoStageSelection  # noqa: E402


def ac_round(x, lag):
    """The autocovariance rounded to one decimal."""
    return np.round(np.mean(x[:, lag:] * x[:, :-lag], axis=1), 1)


def candidates():
    ac1 = partial(MA2.autocov, lag=1)
    ac1.__name__ = 'ac_lag1'
    ac2 = partial(MA2.autocov, lag=2)
    ac2.__name__ = 'ac_lag2'
    r1 = partial(ac_round, lag=1)
    r1.__name__ = 'ac_round1'
    r2 = partial(ac_round, lag=2)
    r2.__name__ = 'ac_round2'
    return ac1, ac2, Gauss.ss_mean, r1, r2


def simulator(discrete=False):
    elfi.new_model()
    if discrete:
        t1 = elfi.Prior('randint', -1, 2, name='t1')
        t2 = elfi.Prior('randint', 0, 2, name='t2')
    else:
        t1 = elfi.Prior(MA2.CustomPrior1, 2, name='t1')
        t2 = elfi.Prior(MA2.CustomPrior2, t1, 1, name='t2')
    y_obs = MA2.MA2(.6, .2, random_state=np.random.RandomState(0))
    return elfi.Simulator(MA2.MA2, t1, t2, observed=y_obs, name='MA2')


def score(sel, n_sim, n_acc, n_closest, batch_size, k=4):
    """run()'s two stages with every intermediate kept; checks that run() agrees."""
    thetas, E = [], []
    E_me, n_me, i_me = np.inf, None, None
    for i, set_ss in enumerate(sel.ss_candidates):
        th = sel._obtain_accepted_thetas(set_ss, n_sim, n_acc, batch_size)
        e = sel._calc_entropy(th, n_acc, k)
        if (e == E_me and n_me > len(set_ss)) or e < E_me:
            E_me, n_me, i_me = e, len(set_ss), i
        thetas.append(np.asarray(th, dtype=np.float64))
        E.append(e)
    closest = thetas[i_me][:n_closest]
    M = [sel._calc_MRSSE(s, closest, th) for s, th in zip(sel.ss_candidates, thetas)]
    chosen = sel.run(n_sim, n_acc=n_acc, n_closest=n_closest, batch_size=batch_size, k=k)
    index = sel.ss_candidates.index(chosen)
    return dict(thetas=np.stack(thetas), entropy=np.array(E), mrsse=np.array(M),
                selected=np.int64(index), closest_from=np.int64(i_me))


def main():
    out = {}
    ac1, ac2, mean, r1, r2 = candidates()
    cases = [
        ('ma2', dict(list_ss=[ac1, ac2, mean]), False, 20000, 2000, 0, None, None),
        ('twice', dict(prepared_ss=[(ac1,), (ac1, ac2), (ac1,)]), False, 5000, 1000, 1, 100, 5),
        ('round', dict(list_ss=[r1, r2]), False, 5000, 1000, 1, 100, 5),
        ('dup', dict(list_ss=[ac1, ac2]), True, 5000, 1000, 1, 100, 5),
    ]
    for name, kw, discrete, n_sim, batch_size, seed, n_acc, n_closest in cases:
        sel = TwoStageSelection(simulator(discrete), 'euclidean', seed=seed, **kw)
        n_acc = n_acc or int(n_sim / 100)
        n_closest = n_closest or int(n_acc / 100)
        for key, val in score(sel, n_sim, n_acc, n_closest, batch_size).items():
            out['{}_{}'.format(name, key)] = val
        out[name + '_config'] = np.array([n_sim, batch_size, seed, n_acc, n_closest])

    rs = np.random.RandomState(7)
    sel = TwoStageSelection(simulator(), 'euclidean', list_ss=[ac1])
    pts, E, M, cfg = [], [], [], []
    for q in range(1, 7):
        for k in (2, 4, 8):           # the reference's query returns a scalar at k = 1
            for n in (k - 1, k, 50):
                if n < 1:
                    continue
                X = rs.randn(n, q)
                if n >= 10:
                    X[5:9] = X[4]          # five equal points
                m = max(1, n // 10)
                with np.errstate(divide='ignore'):
                    E.append(sel._calc_entropy(X, n, k))
                M.append(sel._calc_MRSSE(None, X[:m], X))
                pts.append(X.ravel())
                cfg.append((q, k, n, m))
    out['pts_data'] = np.concatenate(pts)
    out['pts_config'] = np.array(cfg, dtype=np.int64)
    out['pts_entropy'] = np.array(E)
    out['pts_mrsse'] = np.array(M)
    np.savez(os.path.join(HERE, 'diagnostics.npz'), **out)


if __name__ == '__main__':
    main()
