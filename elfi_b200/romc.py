"""Robust optimisation Monte Carlo (ROMC; Ikonomov and Gutmann 2020), the reference's
elfi/methods/inference/romc.py and RomcPosterior (elfi/methods/posteriors.py).

ROMC fixes n1 nuisance seeds; each turns the simulator into a deterministic objective
f_i(theta) = d(theta; seed_i)^2.  Every f_i is minimised (Nelder-Mead), a box is built around each
accepted minimum where f_i < eps, and the boxes are sampled with weight prior(theta) 1[f_i < eps] /
q(theta).  Here all problems advance in lock-step: the Nelder-Mead state machines, the line search
that bounds the boxes, the box draws, the weights and the posterior grid are CUDA kernels
(csrc/romc.cu), and each step evaluates one point of every problem.

Two ways to evaluate the objectives, with one driver:
  * device model (its simulators return device arrays): problem i is row i of one
    ``model.generate(n1, outputs=[discrepancy], with_values=Theta, seed=s)``; a row's Philox stream
    depends only on (s, i), so one launch chain evaluates one point of every problem;
  * any other model: as in the reference, the nuisances are
    ``ss.randint(1, 2**32 - 1).rvs(n1, random_state=seed)`` and problem i is
    ``model.generate(1, with_values=theta_i, seed=nuisance_i)``, one call per point.

Departures from the reference: the Hessian at each minimum is one fixed-step central difference
(see :func:`hessian_points`) instead of numdifftools.Hessian; the vertices of a Nelder-Mead simplex
are ordered by a stable sort (NumPy's order whenever there are no ties, and for p <= 2); the box
draws use Philox (seed, region, point) streams.  Bayesian optimisation (``use_bo=True``), custom
optimisation classes, the plots and multi-rank runs are not provided.
"""
import logging
import math

import numpy as np
import scipy.linalg
import scipy.stats as ss
from scipy import spatial
import torch

from . import device as dev
from . import model as em
from . import ops
from .results import RomcSample
from .samplers import ModelPrior
from .throughput import LazySimulation

logger = logging.getLogger(__name__)

HESSIAN_STEP = 1e-4


def hessian_points(x):
    """The 2 p^2 + 1 points of the fixed-step central-difference Hessian at each row of x (P, p):
    h_i = 1e-4 max(1, |x_i|); x; x +- 2 h_i e_i (diagonal); x +- h_i e_i +- h_j e_j for i < j.
    Returns (points (2 p^2 + 1, P, p), h (P, p))."""
    x = np.asarray(x, dtype=np.float64)
    P, p = x.shape
    h = HESSIAN_STEP * np.maximum(1.0, np.abs(x))
    pts = [x.copy()]
    for i in range(p):
        for s in (2.0, -2.0):
            y = x.copy()
            y[:, i] = x[:, i] + s * h[:, i]
            pts.append(y)
    for i in range(p):
        for j in range(i + 1, p):
            for si, sj in ((1, 1), (1, -1), (-1, 1), (-1, -1)):
                y = x.copy()
                y[:, i] = x[:, i] + si * h[:, i]
                y[:, j] = x[:, j] + sj * h[:, j]
                pts.append(y)
    return np.stack(pts), h


def hessian_from_values(f, h):
    """The Hessians (P, p, p) from f (2 p^2 + 1, P) at :func:`hessian_points`:
    H_ii = (f(x + 2h_i) - 2 f(x) + f(x - 2h_i)) / (4 h_i h_i) and
    H_ij = (f(++) - f(+-) - f(-+) + f(--)) / (4 h_i h_j), evaluated left to right."""
    f = np.asarray(f, dtype=np.float64)
    P, p = h.shape
    H = np.empty((P, p, p))
    f0 = f[0]
    for i in range(p):
        fp, fm = f[1 + 2 * i], f[2 + 2 * i]
        H[:, i, i] = (fp - 2.0 * f0 + fm) / (4.0 * h[:, i] * h[:, i])
    k = 1 + 2 * p
    for i in range(p):
        for j in range(i + 1, p):
            H[:, i, j] = H[:, j, i] = (f[k] - f[k + 1] - f[k + 2] + f[k + 3]) / (4.0 * h[:, i] * h[:, j])
            k += 4
    return H


def find_rotation(hess):
    """RegionConstructor._find_rotation_vector for a stack of Hessians (P, p, p): the eigenvectors
    of each, or the identity where the Hessian is rank deficient or not finite, or the eigenvectors
    are complex, not finite or rank deficient."""
    hess = np.asarray(hess, dtype=np.float64)
    P, p, _ = hess.shape
    eye = np.eye(p)
    finite = np.isfinite(hess).all(axis=(1, 2))
    H = np.where(finite[:, None, None], hess, eye)
    H = np.where((np.linalg.matrix_rank(H) != p)[:, None, None], eye, H)
    out = np.empty_like(H)
    for i in range(P):       # np.linalg.eig of a stack would turn every result complex if one is
        w, v = np.linalg.eig(H[i])
        if np.iscomplexobj(v) or not np.isfinite(np.sum(v)) or np.linalg.matrix_rank(v) < p:
            v = eye
        out[i] = v
    return out


def secure_limits(limits):
    """NDimBoundingBox._secure_limits: widen a side narrower than 0.001 by 0.0005 each way."""
    limits = np.array(limits, dtype=float)
    eps = .001
    for idx in np.ndindex(limits.shape[:-1]):
        if math.isclose(limits[idx][0], limits[idx][1], abs_tol=eps):
            logger.warning('The limits of a dimension of a bounding box are too narrow (<= %s)', eps)
            limits[idx + (0,)] -= eps / 2
            limits[idx + (1,)] += eps / 2
    return limits


def poly2_features(x):
    """PolynomialFeatures(degree=2) of the rows of x (n, p): 1, x_i, then x_i x_j for i <= j."""
    x = np.atleast_2d(np.asarray(x, dtype=np.float64))
    cols = [np.ones(len(x))] + [x[:, i] for i in range(x.shape[1])]
    cols += [x[:, i] * x[:, j] for i in range(x.shape[1]) for j in range(i, x.shape[1])]
    return np.column_stack(cols)


def fit_local_model(x, y):
    """LinearRegression(fit_intercept=False) on poly2_features(x): the minimum-norm least-squares
    coefficients of one region.  scikit-learn 1.9's LinearRegression.fit solves dense X with
    ``scipy.linalg.lstsq(X, y, cond=self.tol)`` (LAPACK gelsd), tol = 1e-6 by default, so singular
    values below 1e-6 of the largest are cut here too."""
    return scipy.linalg.lstsq(poly2_features(x), np.asarray(y, dtype=np.float64), cond=1e-6)[0]


def compute_ess(weights):
    """Effective sample size of unnormalised weights (elfi/methods/utils.py compute_ess)."""
    w = np.atleast_1d(np.asarray(weights, dtype=np.float64))
    if (w < 0).any() or np.sum(w) == 0:
        raise ValueError('Weights must be non-negative and not all zero')
    w = w / np.sum(w)
    return np.square(np.sum(w)) / np.sum(np.square(w))


def _simulators_on_device(model):
    sims = [n for n in model.nodes if model.record(n).cls is em.Simulator]
    if not sims:
        return False
    out = model.generate(2, outputs=sims, seed=1)
    return all(dev.is_device_array(out[n]) or isinstance(out[n], LazySimulation) for n in sims)


class ROMC:
    """Robust optimisation Monte Carlo with the reference's interface (elfi.ROMC).

    ``model`` is the discrepancy node or a model with ``discrepancy_name``; ``bounds`` the
    [(lo, hi), ...] box used to normalise the posterior.  ``device_prior`` is an object whose
    ``logpdf(params)`` gives the joint prior log density of device rows (e.g.
    ``DeviceModelPrior(model)`` or an example's ``DeviceProposal``); device models need one (the
    default is ``DeviceModelPrior(model)``), other models use the host prior density.
    ``parallelize`` is accepted and has no effect: the problems always advance together.

    Starting points are ``prior.rvs(size=n1, random_state=seed)`` as in the reference.  A device
    prior keys its Philox stream from a RandomState, not from an integer, so on a device model the
    seed is passed as ``np.random.RandomState(seed)``; host priors take the seed itself."""

    def __init__(self, model, bounds=None, discrepancy_name=None, output_names=None,
                 custom_optim_class=None, parallelize=False, device_prior=None, **kwargs):
        if custom_optim_class is not None:
            raise NotImplementedError('custom optimisation classes are not supported: the '
                                      'problems are solved by the lock-step device Nelder-Mead')
        if kwargs.get('rank') is not None or kwargs.get('world_size', 1) != 1:
            raise NotImplementedError('ROMC runs on one rank')
        if isinstance(model, em.NodeReference):
            discrepancy_name = model.name
            model = model.model
        if not isinstance(model, em.ElfiModel) or discrepancy_name is None:
            raise ValueError('pass the discrepancy node, or a model and its discrepancy_name')
        if discrepancy_name not in model.nodes:
            raise ValueError('Node {} is not in the model'.format(discrepancy_name))
        self.model = model
        self.discrepancy_name = discrepancy_name
        self.parameter_names = list(model.parameter_names)
        self.prior = ModelPrior(model)
        self.dim = self.prior.dim
        ops._romc_p(self.dim)
        self.bounds = bounds
        self.left_lim = None if bounds is None else np.array([b[0] for b in bounds], dtype=float)
        self.right_lim = None if bounds is None else np.array([b[1] for b in bounds], dtype=float)
        self.on_device = _simulators_on_device(model)
        self.device_prior = device_prior
        if self.on_device and device_prior is None:
            from .priors import DeviceModelPrior
            self.device_prior = DeviceModelPrior(model)
        self.inference_args = {'parallelize': parallelize}
        self.inference_state = {'_has_solved_problems': False, '_has_defined_posterior': False,
                                '_has_drawn_samples': False, '_has_fitted_local_models': False}
        self.samples = self.weights = self.distances = self.result = None
        self.partition = None

    # ---- objectives -----------------------------------------------------------------------
    def _evaluate(self, theta, rows=None):
        """f_i(theta_i) = d^2 for the rows of theta (n1, p), as a device array (n1,).  The host
        path evaluates only `rows` (all by default); the others are 0."""
        n1 = self.n1
        name = self.discrepancy_name
        if self.on_device:
            t = theta if dev.is_device_array(theta) else dev.to_device(np.asarray(theta))
            vals = {pn: t[:, k].contiguous() for k, pn in enumerate(self.parameter_names)}
            d = self.model.generate(n1, outputs=[name], with_values=vals,
                                    seed=self._sim_seed)[name]
            d = (d if dev.is_device_array(d) else dev.to_device(np.asarray(d))).reshape(-1)
            return d * d
        t = dev.to_host(theta) if dev.is_device_array(theta) else np.asarray(theta)
        out = np.zeros(n1)
        for i in (range(n1) if rows is None else np.flatnonzero(rows)):
            params = {pn: np.expand_dims(t[i, k:k + 1], 0)
                      for k, pn in enumerate(self.parameter_names)}
            d = self.model.generate(1, outputs=[name], with_values=params,
                                    seed=int(self.nuisance[i]))[name]
            d = dev.to_host(d) if dev.is_device_array(d) else d
            out[i] = float(np.asarray(d).reshape(-1)[0]) ** 2
        return dev.to_device(out)

    def _evaluate_batches(self, theta, rows=None, cols=None):
        """f at theta (K, n1, p): batch k evaluates theta[k]; a device array (K, n1), or (K, len(cols))
        with only the columns cols of each batch kept."""
        idx = None if cols is None else dev.to_device(np.asarray(cols, dtype=np.int64),
                                                      dtype=torch.int64)
        out = []
        for k in range(theta.shape[0]):
            t = np.ascontiguousarray(theta[k]) if isinstance(theta, np.ndarray) else theta[k]
            f = self._evaluate(t, rows)
            out.append(f if idx is None else f[idx])
        return torch.stack(out)

    def _prior_pdf(self, theta):
        """Joint prior density of the rows of theta (n, p), a device array (n,)."""
        if self.device_prior is not None:
            t = theta if dev.is_device_array(theta) else dev.to_device(np.asarray(theta))
            return self.device_prior.logpdf(t.reshape(-1, self.dim).contiguous()).exp()
        t = dev.to_host(theta) if dev.is_device_array(theta) else np.asarray(theta)
        t = t.reshape(-1, self.dim)
        return dev.to_device(np.array([float(np.reshape(self.prior.pdf(t[i:i + 1]), -1)[0])
                                       for i in range(len(t))]))

    # ---- training ------------------------------------------------------------------------
    def solve_problems(self, n1, use_bo=False, optimizer_args=None, seed=None):
        """Define n1 deterministic problems and minimise each with Nelder-Mead from x0 =
        prior.rvs(size=n1, random_state=seed)[i]; then the Hessian at each solution."""
        if not isinstance(n1, (int, np.integer)) or n1 < 1:
            raise ValueError('n1 must be a positive integer, got {!r}'.format(n1))
        if use_bo:
            raise NotImplementedError('use_bo=True (Bayesian optimisation of the objectives) is not '
                                      'provided; use the gradient-free Nelder-Mead path')
        args = dict(optimizer_args or {})
        method = args.pop('method', 'Nelder-Mead')
        if method != 'Nelder-Mead':
            raise NotImplementedError('only method="Nelder-Mead" is provided, got {!r}'.format(method))
        args.pop('jac', None)         # Nelder-Mead ignores the Jacobian, as scipy does
        opt_seed = args.pop('seed', seed)
        x0 = args.pop('x0', None)
        if args:
            raise ValueError('unknown optimizer_args {}'.format(sorted(args)))
        self.n1 = int(n1)
        self.nuisance = ss.randint(low=1, high=2 ** 32 - 1).rvs(size=self.n1, random_state=seed)
        self._sim_seed = int(np.random.RandomState(seed).randint(2 ** 31)) if seed is None else seed
        if x0 is None:
            # device priors key their Philox streams from a RandomState; host priors take the
            # seed itself, as in the reference
            rs = np.random.RandomState(opt_seed) if self.on_device else opt_seed
            x0 = self.prior.rvs(size=self.n1, random_state=rs)
        x0 = np.asarray(dev.to_host(x0) if dev.is_device_array(x0) else x0, dtype=np.float64)
        x0 = np.broadcast_to(x0.reshape(-1, self.dim) if x0.size != self.dim else x0.reshape(1, -1),
                             (self.n1, self.dim))
        self.x0 = np.ascontiguousarray(x0)
        nm = ops.RomcNelderMead(self.x0)
        while True:
            running = None if self.on_device else \
                dev.to_host(nm.istate[:, 0]) != ops.ROMC_NM_DONE
            if running is not None and not running.any():
                break
            nm.step(self._evaluate(nm.theta, running))
            if running is None and nm.running() == 0:
                break
        self.x_min, self.f_min, self.nit, self.nfev, self.solved = nm.result()
        pts, h = hessian_points(self.x_min)
        f = dev.to_host(self._evaluate_batches(pts, self.solved))
        self.hess = hessian_from_values(f, h)
        self.inference_state['_has_solved_problems'] = True
        self.inference_state['solved'] = self.solved
        self.inference_state['attempted'] = np.ones(self.n1, dtype=bool)

    def compute_eps(self, quantile):
        """The quantile of the optimal distances of the solved problems."""
        self._require('_has_solved_problems', 'solve the optimisation problems first')
        quantile = float(quantile)
        if not 0 <= quantile <= 1:
            raise ValueError('quantile must lie in [0, 1], got {}'.format(quantile))
        return np.quantile(self.f_min[self.solved], quantile)

    def estimate_regions(self, eps_filter, use_surrogate=False, region_args=None, fit_models=True,
                         fit_models_args=None, eps_region=None, eps_cutoff=None):
        """Keep the solutions with f_min < eps_filter, bound each by a box along the eigenvectors
        of its Hessian, optionally fit a local quadratic per box, and define the posterior."""
        self._require('_has_solved_problems', 'You have firstly to solve the optimization problems.')
        if use_surrogate:
            raise NotImplementedError('use_surrogate=True needs the Bayesian-optimisation '
                                      'surrogate, which is not provided')
        region_args = dict(region_args or {})
        eps_cutoff = eps_filter if eps_cutoff is None else eps_cutoff
        eps_region = region_args.get('eps_region', eps_filter if eps_region is None else eps_region)
        self.eps_filter, self.eps_region, self.eps_cutoff = eps_filter, eps_region, eps_cutoff
        self.accepted = self.solved & (self.f_min < eps_filter)
        logger.info('Total solutions: %d, Accepted solutions after filtering: %d',
                    int(self.solved.sum()), int(self.accepted.sum()))
        rot = np.broadcast_to(np.eye(self.dim), (self.n1, self.dim, self.dim)).copy()
        if self.accepted.any():
            rot[self.accepted] = find_rotation(self.hess[self.accepted])
        ls = ops.RomcLineSearch(self.x_min, rot, self.accepted, eps_region,
                                K=region_args.get('K', 10), eta=region_args.get('eta', 1.),
                                rep_lim=region_args.get('rep_lim', 300))
        while ls.running():
            rows = None if self.on_device else \
                (dev.to_host(ls.istate[:, 2]).reshape(2 * self.dim, self.n1) == 0)
            if rows is None:
                f = self._evaluate_batches(ls.theta)
            else:
                f = torch.stack([self._evaluate(ls.theta[k], rows[k]) for k in range(2 * self.dim)])
            ls.step(f)
        idx = np.flatnonzero(self.accepted)
        self.region_problem = idx
        self.limits = secure_limits(ls.limits()[idx])
        self.rotation = rot[idx]
        self.rotation_inv = np.linalg.inv(self.rotation) if len(idx) else self.rotation.copy()
        self.center = self.x_min[idx].copy()
        self.volume = np.prod(-self.limits[:, :, 0] + self.limits[:, :, 1], axis=1)
        self.coef = None
        self.inference_state['_has_fitted_local_models'] = False
        if fit_models:
            args = dict(fit_models_args or {})
            n = int(args.get('nof_samples', 20))
            seed = args.get('seed', self._sim_seed)
            pts, _, _ = self._box_sample(n, seed, with_surrogate=False)
            y = dev.to_host(self._evaluate_regions(pts))
            x = dev.to_host(pts)
            self.local_x, self.local_y = x, y
            self.coef = np.array([fit_local_model(x[r], y[r]) for r in range(len(idx))]).reshape(
                len(idx), 1 + self.dim + self.dim * (self.dim + 1) // 2)
            self.inference_state['_has_fitted_local_models'] = True
        self.partition = None
        self.inference_state['_has_defined_posterior'] = True

    def fit_posterior(self, n1, eps_filter, use_bo=False, quantile=None, optimizer_args=None,
                      region_args=None, fit_models=False, fit_models_args=None, seed=None,
                      eps_region=None, eps_cutoff=None):
        """solve_problems, compute_eps (eps_filter='auto'), estimate_regions."""
        if eps_filter == 'auto' and not isinstance(quantile, (int, float)):
            raise ValueError('eps_filter="auto" needs a quantile')
        self.solve_problems(n1=n1, use_bo=use_bo, optimizer_args=optimizer_args, seed=seed)
        eps_filter = self.compute_eps(float(quantile)) if eps_filter == 'auto' else float(eps_filter)
        self.estimate_regions(eps_filter=eps_filter, use_surrogate=use_bo, region_args=region_args,
                              fit_models=fit_models, fit_models_args=fit_models_args,
                              eps_region=eps_region, eps_cutoff=eps_cutoff)

    def _box_sample(self, n, seed, with_surrogate):
        return ops.romc_box_sample(self.center, self.rotation, self.rotation_inv, self.limits,
                                   self.volume, n, seed,
                                   coef=self.coef if with_surrogate else None)

    def _evaluate_regions(self, pts):
        """f of each region's own problem at pts (R, n, p); a device array (R, n)."""
        R, n = int(pts.shape[0]), int(pts.shape[1])
        full = np.zeros((n, self.n1, self.dim))
        full[:, self.region_problem] = np.transpose(dev.to_host(pts), (1, 0, 2))
        rows = np.zeros(self.n1, dtype=bool)
        rows[self.region_problem] = True
        return self._evaluate_batches(full, rows, self.region_problem).T.contiguous()

    # ---- inference -----------------------------------------------------------------------
    def sample(self, n2, seed=None):
        """n2 weighted draws from every region (RomcPosterior.sample)."""
        self._require('_has_defined_posterior', 'You must train first')
        if seed is None:
            seed = int(np.random.randint(2 ** 31))
        local = self.coef is not None
        pts, q, surr = self._box_sample(int(n2), seed, with_surrogate=local)
        dist = surr if local else self._evaluate_regions(pts)
        pr = self._prior_pdf(pts.reshape(-1, self.dim)).reshape(tuple(q.shape))
        w = ops.romc_weights(dist, pr, q, self.eps_cutoff)
        self.samples = dev.to_host(pts)
        self.weights = dev.to_host(w)
        self.distances = dev.to_host(dist).reshape(-1)
        self.inference_state['_has_drawn_samples'] = True
        self.result = self.extract_result()

    def eval_unnorm_posterior(self, theta):
        """The unnormalised posterior at the rows of theta (M, p)."""
        self._require('_has_defined_posterior', 'You must train first')
        theta = np.asarray(theta, dtype=np.float64)
        if theta.ndim != 2 or theta.shape[1] != self.dim:
            raise ValueError('theta must be (M, {})'.format(self.dim))
        pr = self._prior_pdf(theta)
        if self.coef is not None:
            out = ops.romc_posterior_unnorm(theta, pr, self.eps_cutoff, self.center,
                                            self.rotation_inv, self.limits, self.coef)
        else:
            M = len(theta)
            rows = np.zeros(self.n1, dtype=bool)
            rows[self.region_problem] = True
            full = np.broadcast_to(theta[:, None, :], (M, self.n1, self.dim))
            f = self._evaluate_batches(full, rows, self.region_problem)
            out = ops.romc_posterior_unnorm(theta, pr, self.eps_cutoff, fvals=f)
        return dev.to_host(out)

    def _approximate_partition(self, nof_points=30):
        if self.dim > 2:
            raise ValueError('the partition function is approximated for 1 and 2 dimensions only')
        vol_per_point = np.prod((self.right_lim - self.left_lim) / nof_points)
        axes = [np.linspace(self.left_lim[i], self.right_lim[i], nof_points)
                for i in range(self.dim)]
        grid = np.array([[a] for a in axes[0]]) if self.dim == 1 else \
            np.array([[a, b] for a in axes[0] for b in axes[1]])
        self.partition = np.sum(self.eval_unnorm_posterior(grid) * vol_per_point)
        return self.partition

    def eval_posterior(self, theta):
        """The posterior at the rows of theta, normalised on a 30-point grid per axis of the
        bounds (1 and 2 dimensions)."""
        self._require('_has_defined_posterior', 'You must train first')
        if self.bounds is None:
            raise ValueError('You have to set the bounds in order to approximate the partition '
                             'function')
        partition = self.partition if self.partition is not None else self._approximate_partition()
        return self.eval_unnorm_posterior(theta) / partition

    def compute_expectation(self, h):
        """sum(h(samples) w) / sum(w) over the weighted draws."""
        self._require('_has_drawn_samples', 'Draw samples first')
        return np.sum(h(self.samples) * self.weights) / np.sum(self.weights)

    def compute_ess(self):
        self._require('_has_drawn_samples', 'Draw samples first')
        return compute_ess(self.result.weights)

    def compute_divergence(self, gt_posterior, bounds=None, step=0.1, distance='Jensen-Shannon'):
        """Jensen-Shannon distance or KL divergence to gt_posterior on a grid (1 and 2 dims)."""
        self._require('_has_defined_posterior', 'You must train first')
        if distance not in ('Jensen-Shannon', 'KL-Divergence'):
            raise ValueError('distance must be "Jensen-Shannon" or "KL-Divergence"')
        if bounds is None and self.bounds is None:
            raise ValueError("You have to define the prior's limits in order to compute the "
                             "divergence")
        limits = [(self.left_lim[i], self.right_lim[i]) for i in range(len(self.left_lim))]
        if len(limits) > 2:
            logger.info('Computational approximation of KL Divergence on D > 2 is intractable.')
            return None
        axes = [np.linspace(lo, hi, int((hi - lo) / step)) for lo, hi in limits]
        if len(limits) == 1:
            x = np.expand_dims(axes[0], -1)
        else:
            gx, gy = np.meshgrid(*axes)
            x = np.stack((gx.flatten(), gy.flatten()), -1)
        p_points = np.squeeze(self.eval_posterior(x))
        q_points = np.squeeze(gt_posterior(x))
        if distance == 'KL-Divergence':
            return ss.entropy(p_points, q_points)
        return spatial.distance.jensenshannon(p_points, q_points)

    def extract_result(self):
        """The weighted draws as a RomcSample (parameters and discrepancies flattened region by
        region)."""
        if self.samples is None:
            raise ValueError('Nothing to extract')
        outputs = {name: self.samples[:, :, i].flatten()
                   for i, name in enumerate(self.parameter_names)}
        outputs[self.discrepancy_name] = self.distances.flatten()
        return RomcSample(method_name='ROMC', outputs=outputs,
                          parameter_names=self.parameter_names,
                          discrepancy_name=self.discrepancy_name, weights=self.weights.flatten())

    def visualize_region(self, *args, **kwargs):
        raise NotImplementedError('plots are not provided')

    def distance_hist(self, *args, **kwargs):
        raise NotImplementedError('plots are not provided')

    def _require(self, flag, msg):
        if not self.inference_state.get(flag):
            raise ValueError(msg)
