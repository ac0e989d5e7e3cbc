"""Golden fixtures for the Lotka-Volterra example, from the UNMODIFIED reference (elfi-dev/elfi, the
checkout named by ELFI_REFERENCE_ROOT).

    ELFI_REFERENCE_ROOT=<checkout> python tests/golden/gen_golden_lotka_volterra.py

* lv_draws.npz     -- elfi.examples.lotka_volterra.lotka_volterra for seeded RandomStates: the
                      default truth; a mixed batch in which the predators die out mid-run, start at
                      0 (the ramp to a fictitious event at time_end) or both species start at 0
                      (infinite times, the null reaction); observation noise that drives counts
                      negative (truncation toward zero); and, with return_full, a row of more than
                      20000 steps (the float64 switch of the event arrays).  Of return_full's
                      event arrays only the shape, dtype, SHA-256 and last events are kept.
* lv_summaries.npz -- the reference's nine summaries of those draws and of crafted inputs
                      (constant series, n_obs = 3, large counts, non-default mu / std).
* lv_rejection.npz -- Rejection(lotka_volterra.get_model(seed_obs=..., time_end=...)['d'], ...)
                      .sample(...), with a shortened time_end so that prior draws stay cheap.
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

from ref_shim import import_reference  # noqa: E402

elfi = import_reference()
from elfi.examples import lotka_volterra as lv  # noqa: E402

TRUTH = [1.0, 0.005, 0.6, 50, 100, 0.]
# (r1, r2, r3, prey0, predator0, sigma): the truth, predators dying out, predators starting at 0,
# both species at 0, a prey-free start, fractional initial counts
MIXED = np.array([[1.0, 0.005, 0.6, 50, 100, 0.],
                  [0.1, 0.02, 1.5, 30.0, 12.0, 0.],
                  [0.5, 0.05, 3.0, 10.0, 4.0, 0.],
                  [1.0, 0.005, 0.6, 40.0, 0.5, 0.],
                  [0.7, 0.005, 0.6, 0.3, 0.2, 0.],
                  [1.0, 0.005, 0.6, 0.0, 30.0, 0.],
                  [2.0, 0.001, 0.2, 20.7, 15.99, 0.]])
NOISY = np.array([[1.0, 0.005, 0.6, 3.0, 2.0, 10.0],
                  [1.0, 0.005, 0.6, 50, 100, 10.0],
                  [0.3, 0.01, 1.0, 1.0, 1.0, 25.0]])
LONG = dict(r1=1.0, r2=0.001, r3=1.0, prey_init=1000, predator_init=1000, time_end=8.0, n_obs=20)
REJECTION = dict(seed_obs=7, time_end=0.5, batch_size=20, seed=3, n=10, quantile=0.1)


def save(name, **arrays):
    np.savez_compressed(os.path.join(HERE, name + '.npz'), **arrays)
    print('wrote', name, {k: np.shape(v) for k, v in arrays.items()})


def summaries(x, **kw):
    with np.errstate(all='ignore'):
        return np.column_stack([
            lv.stock_mean(x, species=0, **kw), lv.stock_mean(x, species=1, **kw),
            lv.stock_log_variance(x, species=0, **kw), lv.stock_log_variance(x, species=1, **kw),
            lv.stock_autocorr(x, species=0, lag=1, **kw), lv.stock_autocorr(x, species=1, lag=1, **kw),
            lv.stock_autocorr(x, species=0, lag=2, **kw), lv.stock_autocorr(x, species=1, lag=2, **kw),
            lv.stock_crosscorr(x, **kw)])


def digest(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), dtype=np.uint8)


def keep_full(out, name, stock, times):
    """The shape, dtype, SHA-256 and last 10 events of return_full's event arrays."""
    out[name + '_stock_shape'] = np.array(stock.shape)
    out[name + '_stock_dtype'] = np.array(str(stock.dtype))
    out[name + '_stock_sha'] = digest(stock)
    out[name + '_times_sha'] = digest(times)
    out[name + '_stock_tail'] = stock[:, -10:]
    out[name + '_times_tail'] = times[:, -10:]


def main():
    out = {}
    out['truth'] = lv.lotka_volterra(*TRUTH, n_obs=50, batch_size=3,
                                     random_state=np.random.RandomState(1))
    with np.errstate(all='ignore'):
        full = lv.lotka_volterra(*MIXED.T, n_obs=30, batch_size=len(MIXED),
                                 random_state=np.random.RandomState(2), return_full=True)
    out['mixed_prm'] = MIXED
    out['mixed'] = full[0]
    keep_full(out, 'mixed', full[2], full[3])
    out['noisy_prm'] = NOISY
    out['noisy'] = lv.lotka_volterra(*NOISY.T, n_obs=25, batch_size=len(NOISY),
                                     random_state=np.random.RandomState(3))
    a = LONG
    so, to, stock, times = lv.lotka_volterra(a['r1'], a['r2'], a['r3'], a['prey_init'],
                                             a['predator_init'], n_obs=a['n_obs'],
                                             time_end=a['time_end'],
                                             random_state=np.random.RandomState(4), return_full=True)
    out['long'], out['long_times_out'] = so, to
    keep_full(out, 'long', stock, times)
    save('lv_draws', **out)

    s = {}
    for name in ('truth', 'mixed', 'noisy', 'long'):
        s[name] = summaries(out[name])
    rs = np.random.RandomState(5)
    crafted = {
        'constant': np.tile(np.array([[[7, 3]]], dtype=np.int32), (2, 12, 1)),
        'n3': rs.randint(-5, 200, (4, 3, 2)).astype(np.int32),
        'large': rs.randint(-2 ** 31, 2 ** 31 - 1, (3, 40, 2)).astype(np.int32),
        'n128': rs.randint(0, 500, (3, 128, 2)).astype(np.int32),
    }
    crafted['constant'][1, :, 0] = np.arange(12)
    for name, x in crafted.items():
        s['x_' + name] = x
        s[name] = summaries(x)
    s['truth_scaled'] = summaries(out['truth'], mu=3.5, std=0.25)
    save('lv_summaries', **s)

    r = REJECTION
    m = lv.get_model(seed_obs=r['seed_obs'], time_end=r['time_end'])
    res = elfi.Rejection(m['d'], batch_size=r['batch_size'], seed=r['seed']).sample(
        r['n'], quantile=r['quantile'])
    res_out = dict(n_sim=res.n_sim, threshold=res.threshold, d=res.discrepancies,
                   observed=np.asarray(m.observed['LV']))
    for k, v in res.samples.items():
        res_out['out_' + k] = np.asarray(v)
    save('lv_rejection', **res_out)


if __name__ == '__main__':
    main()
