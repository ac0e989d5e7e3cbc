"""Golden fixtures for ROMC from the UNMODIFIED reference (elfi-dev/elfi, the checkout named by
ELFI_REFERENCE_ROOT).

    ELFI_REFERENCE_ROOT=<checkout> python tests/golden/gen_golden_romc.py

numdifftools is not installed, so numdifftools.Hessian is replaced here -- and only here -- by the
fixed-step central difference elfi_b200 uses (h_i = 1e-4 max(1, |x_i|); the +-2h stencil on the
diagonal and the four-point stencil off it), written out independently below.  scipy.optimize.minimize
is wrapped to record nit and nfev, and NDimBoundingBox.sample to record the points the local
surrogates are fitted on.

* romc.npz, for the cases 'oned' (tests/romc_cases.py one_d_model, n1 = 100, seed = 21,
  eps_filter = 0.75, local models, n2 = 30) and 'ma2' (the host MA2 model, n_obs = 50,
  true_params [.6, .2], seed_obs = 3; n1 = 20, seed = 5, eps_filter the 0.6 quantile of the optimal
  distances, local models, n2 = 10): <case>_nuisance, _x0, _x_min, _f_min, _success, _nit, _nfev,
  _hess (solved problems), _accepted, _rotation, _center, _limits (regions), _fit_x, _fit_y, _coef
  (local surrogates), _samples, _weights, _distances, _eps.  The surrogate fitting points are drawn
  from NumPy's global generator unseeded, as the reference draws them, and stored.
* romc_fits.npz -- OptimisationProblem.fit_local_surrogate (PolynomialFeatures(degree=2) and
  LinearRegression(fit_intercept=False)) on crafted boxes where the fit is ill-conditioned or
  underdetermined: p = 1 and 2 boxes as narrow as _secure_limits leaves them (width 1e-3), p = 3 with
  mixed widths, and p = 5 (21 coefficients from 20 points), wide and narrow.  Per case <case>_x (the
  20 points), _y (the objective there) and _coef.  Run with the argument 'fits' to write only this.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from ref_shim import import_reference  # noqa: E402

elfi = import_reference()
import elfi.methods.inference.romc as rr  # noqa: E402
from elfi.examples import ma2  # noqa: E402

import romc_cases  # noqa: E402


class FixedHessian:
    def __init__(self, f):
        self.f = f

    def __call__(self, x):
        x = np.asarray(x, dtype=float)
        p = len(x)
        h = 1e-4 * np.maximum(1.0, np.abs(x))
        f0 = self.f(x.copy())
        H = np.empty((p, p))

        def at(steps):
            y = x.copy()
            for i, s in steps:
                y[i] = x[i] + s * h[i]
            return self.f(y)
        for i in range(p):
            H[i, i] = (at([(i, 2.0)]) - 2.0 * f0 + at([(i, -2.0)])) / (4.0 * h[i] * h[i])
        for i in range(p):
            for j in range(i + 1, p):
                H[i, j] = H[j, i] = (at([(i, 1), (j, 1)]) - at([(i, 1), (j, -1)])
                                     - at([(i, -1), (j, 1)]) + at([(i, -1), (j, -1)])) / \
                    (4.0 * h[i] * h[j])
        return H


RESULTS, FITS = [], []
_minimize = rr.optim.minimize


def recording_minimize(*args, **kwargs):
    res = _minimize(*args, **kwargs)
    RESULTS.append(res)
    return res


_sample = rr.NDimBoundingBox.sample


def recording_sample(self, n2, seed=None):
    x = _sample(self, n2, seed)
    FITS.append(x)
    return x


rr.nd.Hessian = FixedHessian
rr.optim.minimize = recording_minimize


def run(name, romc, n1, seed, eps, n2, nof_samples=20):
    RESULTS.clear()
    FITS.clear()
    romc.solve_problems(n1=n1, seed=seed)
    if isinstance(eps, float) and eps < 0:
        eps = float(romc.compute_eps(-eps))
    rr.NDimBoundingBox.sample = recording_sample
    try:
        romc.estimate_regions(eps_filter=eps, fit_models=True,
                              fit_models_args={'nof_samples': nof_samples})
    finally:
        rr.NDimBoundingBox.sample = _sample
    np.random.seed(1)
    romc.sample(n2=n2)
    probs = romc.optim_problems
    out = {'nuisance': np.array([pr.nuisance for pr in probs], dtype=np.int64),
           'x0': np.array([np.atleast_1d(pr.initial_point if pr.initial_point is not None else
                                         np.nan) for pr in probs], dtype=float),
           'x_min': np.array([r.x for r in RESULTS]).reshape(n1, -1),
           'f_min': np.array([r.fun for r in RESULTS]),
           'success': np.array([r.success for r in RESULTS]),
           'nit': np.array([r.nit for r in RESULTS]),
           'nfev': np.array([r.nfev for r in RESULTS]),
           'hess': np.array([pr.result.hess_appr for pr in probs if pr.state['solved']]),
           'accepted': np.array(romc.inference_state['accepted']),
           'eps': np.float64(eps)}
    regs = [pr.regions[0] for pr in probs if pr.state['region']]
    out['rotation'] = np.array([r.rotation for r in regs])
    out['center'] = np.array([r.center for r in regs])
    out['limits'] = np.array([r.limits for r in regs])
    surr = [pr.local_surrogates[0].keywords['model_scikit'] for pr in probs if pr.state['region']]
    objs = [pr.objective for pr in probs if pr.state['region']]
    out['fit_x'] = np.array(FITS)
    out['fit_y'] = np.array([[f(xx) for xx in x] for f, x in zip(objs, FITS)])
    out['coef'] = np.array([m.named_steps['linear'].coef_ for m in surr])
    out['samples'] = np.asarray(romc.samples)
    out['weights'] = np.asarray(romc.weights)
    out['distances'] = np.asarray(romc.distances)
    print(name, {k: np.shape(v) for k, v in out.items()})
    return {name + '_' + k: v for k, v in out.items()}


def fit_objective(x):
    x = np.asarray(x, dtype=float)
    return float(np.sum((np.arange(1, len(x) + 1) * (x - 0.3)) ** 2) + 0.5 * np.sin(np.sum(x)))


def fit_cases():
    rs = np.random.RandomState(7)

    def rot(p):
        return np.linalg.qr(rs.randn(p, p))[0]
    c45 = np.cos(np.radians(45))
    cases = {
        'p1_narrow': (np.eye(1), np.array([0.7]), np.array([[-5e-4, 5e-4]])),
        'p2_narrow': (np.array([[c45, -c45], [c45, c45]]), np.array([0.2, -0.4]),
                      np.array([[-1e-3, 1e-3], [-5e-4, 5e-4]])),
        'p3_mixed': (rot(3), rs.randn(3), np.array([[-5e-4, 5e-4], [-.3, .2], [-1., 1.]])),
        'p5_wide': (rot(5), rs.randn(5), np.column_stack([-rs.uniform(.2, .6, 5),
                                                          rs.uniform(.2, .6, 5)])),
        'p5_narrow': (rot(5), rs.randn(5), np.tile([-5e-4, 5e-4], (5, 1))),
    }
    arrays = {}
    rr.NDimBoundingBox.sample = recording_sample
    try:
        for k, (name, (R, c, lim)) in enumerate(cases.items()):
            FITS.clear()
            prob = rr.OptimisationProblem(0, 1, ['x%d' % i for i in range(len(c))], 'd',
                                          fit_objective, len(c), None, 1, None)
            prob.regions = [rr.NDimBoundingBox(R, c, lim)]
            np.random.seed(100 + k)
            prob.fit_local_surrogate(nof_samples=20)
            x = FITS[0]
            arrays[name + '_x'] = x
            arrays[name + '_y'] = np.array([fit_objective(xx) for xx in x])
            arrays[name + '_coef'] = \
                prob.local_surrogates[0].keywords['model_scikit'].named_steps['linear'].coef_
    finally:
        rr.NDimBoundingBox.sample = _sample
    np.savez(os.path.join(HERE, 'romc_fits.npz'), **arrays)
    print('wrote romc_fits.npz', {k: np.shape(v) for k, v in arrays.items()})


def main():
    fit_cases()
    if sys.argv[1:] == ['fits']:
        return
    arrays = {}
    m, dname = romc_cases.one_d_model(elfi)
    arrays.update(run('oned', elfi.ROMC(m[dname], [(-2.5, 2.5)]), 100, 21, .75, 30))
    m = ma2.get_model(n_obs=50, true_params=[.6, .2], seed_obs=3)
    arrays.update(run('ma2', elfi.ROMC(m['d'], [(-2, 2), (-1, 1)]), 20, 5, -0.6, 10))
    np.savez(os.path.join(HERE, 'romc.npz'), **arrays)
    print('wrote romc.npz')


if __name__ == '__main__':
    main()
