"""Golden fixtures for the Ricker example, from the UNMODIFIED reference (elfi-dev/elfi, the checkout
named by ELFI_REFERENCE_ROOT).

    ELFI_REFERENCE_ROOT=<checkout> python tests/golden/gen_golden_ricker.py

* ricker_draws.npz     -- elfi.examples.ricker.stochastic_ricker for a seeded RandomState over a
                          parameter grid with extinct rows (the stock underflows to 0) and Poisson
                          rates up to ~1e10, and ricker (the deterministic map) over log rates from
                          0.5 (a fixed point) to 12 (extinction) and two initial stocks.
* ricker_summaries.npz -- np.mean, np.var (axis=1) and ricker.num_zeros of those draws, and
                          ricker.chi_squared of them against observed summaries taken from a row,
                          from a row without zeros (#0 = 0: inf and NaN terms), from the row with
                          the most zeros, and the summaries of an extinct series (mean and variance
                          0: inf and NaN terms).
* ricker_rejection.npz -- Rejection(ricker.get_model(seed_obs=...)['d'], ...).sample(...) for the
                          stochastic and the deterministic model.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

from ref_shim import import_reference  # noqa: E402

elfi = import_reference()
from elfi.examples import ricker  # noqa: E402

# (log_rate, std, scale): the default truth, calm, noisy, boom-and-bust with extinction and rates
# near 1e10, a fixed point without noise, heavy noise at a low rate
STOCH_PRM = np.array([[3.8, 0.3, 10.], [2., 0.1, 50.], [6., 1., 1.], [20., 0.5, 60.],
                      [1., 0., 5.], [0.5, 2., 3.], [12., 0.2, 100.]])
DET_RATES = np.array([0.5, 2., 3.8, 6., 12.])
REJECTION = {'stochastic': dict(seed_obs=7, batch_size=20, seed=3, n=30),
             'deterministic': dict(seed_obs=7, batch_size=20, seed=3, n=30)}


def save(name, **arrays):
    np.savez(os.path.join(HERE, name + '.npz'), **arrays)
    print('wrote', name, {k: np.shape(v) for k, v in arrays.items()})


def summaries(y):
    return np.mean(y, axis=1), np.var(y, axis=1), ricker.num_zeros(y)


def main():
    ys = ricker.stochastic_ricker(*STOCH_PRM.T, n_obs=30, batch_size=len(STOCH_PRM),
                                  random_state=np.random.RandomState(3))
    yd1 = ricker.ricker(DET_RATES, n_obs=40, batch_size=len(DET_RATES))
    yd2 = ricker.ricker(DET_RATES, stock_init=0.25, n_obs=40, batch_size=len(DET_RATES))
    save('ricker_draws', stoch_prm=STOCH_PRM, stoch_y=ys, det_rates=DET_RATES, det_y1=yd1,
         det_y2=yd2)

    out = {}
    for name, y in (('stoch', ys), ('det', yd1)):
        s = summaries(y)
        out[name + '_mean'], out[name + '_var'], out[name + '_zeros'] = s
        nz = int(np.argmin(s[2]))          # a row without zeros
        ext = int(np.argmax(s[2]))         # the row with the most zeros
        for tag, row in (('row0', 0), ('nozero', nz), ('mostzeros', ext), ('extinct', None)):
            if row is None:
                obs = summaries(np.zeros((1, y.shape[1])))
            else:
                obs = tuple(v[row:row + 1] for v in s)
            with np.errstate(divide='ignore', invalid='ignore'):
                out['{}_chi_{}'.format(name, tag)] = ricker.chi_squared(*s, observed=obs)
            out['{}_obs_{}'.format(name, tag)] = np.array([v[0] for v in obs], dtype=np.float64)
    save('ricker_summaries', **out)

    res_out = {}
    for variant, a in REJECTION.items():
        m = ricker.get_model(seed_obs=a['seed_obs'], stochastic=variant == 'stochastic')
        res = elfi.Rejection(m['d'], batch_size=a['batch_size'], seed=a['seed']).sample(a['n'])
        res_out[variant + '_n_sim'] = res.n_sim
        res_out[variant + '_threshold'] = res.threshold
        res_out[variant + '_d'] = res.discrepancies
        res_out[variant + '_observed'] = np.asarray(m.observed['Ricker'])
        for k, v in res.samples.items():
            res_out['{}_out_{}'.format(variant, k)] = np.asarray(v)
    save('ricker_rejection', **res_out)


if __name__ == '__main__':
    main()
