"""BOLFI on the device: GP surrogate, LCBSC acquisition, Bayesian optimisation loop.

Mirrors (file:line in elfi-dev/elfi):
  GPyRegression          elfi/methods/bo/gpy_regression.py:15-364   (duck type used by acquisition
                         and posterior code: input_dim, bounds, parameter_names, X, Y, noise,
                         n_evidence, is_sampling, predict, predict_mean, predictive_gradients,
                         predictive_gradient_mean, update, optimize, copy)
  AcquisitionBase, LCBSC elfi/methods/bo/acquisition.py:16-301
  minimize, CostFunction elfi/methods/bo/utils.py:40-164
  BayesianOptimization, BOLFI.fit/extract_posterior   elfi/methods/inference/bolfi.py:26-462
  BolfiPosterior (logpdf / pdf core)                  elfi/methods/posteriors.py:21-189

The GP arithmetic (Gram, Cholesky, inverse factor, predict, gradients, LCBSC) runs in gp.cu.
Kernel: RBF + Bias with the reference's default hyper-parameter heuristics
(gpy_regression.py:255-264).  Hyper-parameter optimisation: GPy (SCG on the marginal likelihood
with Gamma priors) is not available to pin against -> `optimize()` maximises the same objective
(log marginal likelihood + Gamma log-priors) with L-BFGS-B on log-parameters; PARITY UNPINNED.
"""
import copy
import logging
import threading
from math import ceil

import numpy as np
import scipy.optimize
import scipy.stats as ss
import torch

from . import _lib
from . import device as dev
from . import mcmc
from .model import get_sub_seed
from .results import BolfiSample, OptimizationResult
from .samplers import ModelPrior, ParameterInference, resolve_sigmas

logger = logging.getLogger(__name__)

HYPER_LOG_RANGE = np.log(1e3)   # optimize(): search box half-width in log space

JITTER = 1e-8   # GPy's exact Gaussian inference adds 1e-8 to the diagonal


class GPyRegression:
    """GP regression with an RBF + Bias kernel and Gaussian noise, fitted on the device.

    Named after the reference class it stands in for; no GPy involved."""

    def __init__(self, parameter_names=None, bounds=None, optimizer="lbfgsb", max_opt_iters=50,
                 gp=None, incremental=True, **gp_params):
        """`incremental=True` (default): new evidence extends the Cholesky factor by a rank-b
        update (O(b n^2), 3 small launches) instead of a refit whenever the hyper-parameters and
        the padded size are unchanged; equal to a refit to ~1e-7 (the reference rebuilds the GP on
        every update, gpy_regression.py:286-315).  `incremental=False` refits every time."""
        if not (parameter_names is None or isinstance(parameter_names, (list, tuple))):
            raise ValueError('`parameter_names` must be a list of strings')
        self.parameter_names = parameter_names
        self.input_dim = 1 if parameter_names is None else len(parameter_names)
        self.bounds = self._bounds_in_parameter_order(bounds)
        self.gp_params, self.optimizer, self.max_opt_iters = gp_params, optimizer, max_opt_iters
        self.incremental = bool(incremental)
        self._X = None          # host (n, p)
        self._Y = None          # host (n, 1)
        self._hyper = None      # dict(kernel_var, lengthscale, bias_var, noise_var)
        self._priors = None     # Gamma prior (a, b) per hyper-parameter
        self._factor = None     # device tensors of the current fit
        self.is_sampling = False   # duck-type attribute (gpy_regression.py:64); no cached path here

    def _bounds_in_parameter_order(self, bounds):
        """{name: (lower, upper)} -> [(lower, upper)] in the order of the parameter names; the
        unit box (with a warning) when no bounds are given."""
        if bounds is None:
            logger.warning('No parameter bounds given: using [0, 1] for every parameter.')
            return [(0, 1)] * self.input_dim
        if len(bounds) != self.input_dim:
            raise ValueError('{} bounds were given for {} parameters'.format(len(bounds),
                                                                             self.input_dim))
        if not isinstance(bounds, dict):
            raise ValueError('`bounds` must be a dictionary {parameter name: (lower, upper)}')
        if self.input_dim == 1:
            return list(bounds.values())
        return [bounds[name] for name in self.parameter_names]

    # ---- data / state ---------------------------------------------------------------------
    @property
    def n_evidence(self):
        return 0 if self._X is None else len(self._X)

    @property
    def X(self):
        return self._X

    @property
    def Y(self):
        return self._Y

    @property
    def noise(self):
        return self._hyper['noise_var']

    @property
    def hyperparameters(self):
        return dict(self._hyper)

    def _default_hyper(self, x, y):
        """gpy_regression.py:242-284.  The reference's default kernel is GPy's RBF + Bias with
        GPy's own initial values (variance = lengthscale = bias variance = 1); the heuristics from
        the bounds and the first data only parameterise the Gamma priors (and the noise variance,
        :254), so until the first `optimize()` the GP runs on the unit values.  The `gp_params`
        entries 'kernel_var' / 'lengthscale' / 'bias_var' stand in for the reference's
        ``gp_params['kernel']`` (a GPy object, not constructible here)."""
        length_scale = (np.max(self.bounds) - np.min(self.bounds)) / 3.
        kernel_var = (np.max(y) / 3.) ** 2.
        bias_var = kernel_var / 4.
        noise_var = self.gp_params.get('noise_var') or np.max(y) ** 2. / 100.
        self._hyper = dict(kernel_var=1.0, lengthscale=1.0, bias_var=1.0,
                           noise_var=float(noise_var))
        for k in ('kernel_var', 'lengthscale', 'bias_var'):
            if k in self.gp_params and self.gp_params[k] is not None:
                self._hyper[k] = float(self.gp_params[k])
        # Gamma.from_EV(E, V) with E = V = value -> shape a = E^2/V = E, rate b = E/V = 1
        self._priors = {'lengthscale': (length_scale, 1.0), 'kernel_var': (kernel_var, 1.0),
                        'bias_var': (bias_var, 1.0)}
        # centre of the optimiser's search box: the prior means
        self._hyper_anchor = dict(kernel_var=float(kernel_var), lengthscale=float(length_scale),
                                  bias_var=float(bias_var), noise_var=float(noise_var))

    def update(self, x, y, optimize=False):
        """Append evidence and refit (the reference rebuilds the GP on every update, 286-315)."""
        x = np.asarray(dev.to_host(x), dtype=np.float64).reshape((-1, self.input_dim))
        y = np.asarray(dev.to_host(y), dtype=np.float64).reshape((-1, 1))
        if self._X is None:
            self._default_hyper(x, y)
            self._X, self._Y = x, y
        else:
            self._X = np.r_[self._X, x]
            self._Y = np.r_[self._Y, y]
        if not (self.incremental and self._append(x, y)):
            self._fit()
        if optimize:
            self.optimize()

    def _append(self, x_new, y_new):
        """Rank-b update of the factor for b appended points (SURVEY.md section 8f, N3).
        With T = W K(X, x_new) (whitened new points), S = cov(x_new, x_new) + noise I = L22 L22^T:
            L' = [[L, 0], [T, L22]],   W' = L'^-1 = [[W, 0], [-L22^-1 T W, L22^-1]],
            alpha' = W'^T W' y'.
        Only T, T W and the b x b block come from the device (whiten / apply_wt / cross_cov);
        the b x n rows are assembled on the host and written into the padded buffers.
        Returns False when a refit is needed instead (no factor yet, other hyper-parameters, the
        padded size would change, or the new block is not positive definite)."""
        f = self._factor
        if f is None or f.get('hyper') != self._hyper:
            return False
        n, b = f['n'], len(x_new)
        if n + b > f['n_pad'] or n + b != len(self._X):
            return False
        noise = self._hyper['noise_var'] + JITTER
        xq, T = self.whiten(x_new)
        TW = dev.empty((b, n))
        _lib.call('elfi_b200_gp_apply_wt_f64', dev.context(), dev.ptr(T), n, b, dev.ptr(f['U']),
                  f['n_pad'], n, dev.ptr(TW), n, dev.stream_ptr())
        S = dev.to_host(self.cross_covariance((xq, T), (xq, T))) + noise * np.eye(b)
        try:
            L22 = np.linalg.cholesky(0.5 * (S + S.T))
        except np.linalg.LinAlgError:
            return False
        L22inv = np.linalg.inv(L22)
        TW_h = dev.to_host(TW)
        rows = -L22inv @ TW_h                                   # new rows of W (left block)
        y_old = self._Y[:n].ravel()
        z2 = L22inv @ (np.asarray(y_new, dtype=float).ravel() - TW_h @ y_old)
        alpha = np.concatenate([dev.to_host(f['alpha']) + rows.T @ z2, L22inv.T @ z2])
        end = n + b
        f['W'][n:end, :n] = dev.to_device(rows)
        f['W'][n:end, n:end] = dev.to_device(L22inv)
        f['U'][:n, n:end] = dev.to_device(np.ascontiguousarray(rows.T))
        f['U'][n:end, n:end] = dev.to_device(np.ascontiguousarray(L22inv.T))
        f['L'][n:end, :n] = T
        f['L'][n:end, n:end] = dev.to_device(L22)
        f.update(X=dev.to_device(self._X), y=dev.to_device(self._Y.reshape(-1)), n=end,
                 alpha=dev.to_device(alpha))
        return True

    def _fit(self, hyper=None):
        h = hyper or self._hyper
        n, p = self._X.shape
        n_pad = int(_lib.load().elfi_b200_gp_padded_size(n))
        Xd = dev.to_device(self._X)
        yd = dev.to_device(self._Y.reshape(-1))
        f = self._factor
        if f is None or f['n_pad'] != n_pad:
            f = dict(n_pad=n_pad, L=dev.empty((n_pad, n_pad)), W=dev.empty((n_pad, n_pad)),
                     U=dev.empty((n_pad, n_pad)))
        f.update(X=Xd, y=yd, n=n, alpha=dev.empty((n,)),
                 info=dev.zeros((1,), dtype=torch.int32))
        _lib.call('elfi_b200_gp_fit_f64', dev.context(), dev.ptr(Xd), p, dev.ptr(yd), n, p,
                  h['kernel_var'], h['lengthscale'], h['bias_var'], h['noise_var'] + JITTER,
                  dev.ptr(f['L']), dev.ptr(f['W']), dev.ptr(f['U']), n_pad, dev.ptr(f['alpha']),
                  dev.ptr(f['info']), dev.stream_ptr())
        info = int(f['info'].item())
        if info != 0:
            raise np.linalg.LinAlgError('Cholesky failed: non-positive pivot at {}'.format(info - 1))
        f['hyper'] = dict(h)
        self._factor = f
        return f

    # ---- prediction -----------------------------------------------------------------------
    def predict(self, x, noiseless=False):
        """GP mean and variance at x -> ((m, 1), (m, 1)) host arrays (gpy_regression.py:98-149)."""
        x = np.asanyarray(dev.to_host(x), dtype=np.float64).reshape((-1, self.input_dim))
        if self._factor is None:
            return np.zeros((x.shape[0], 1)), np.ones((x.shape[0], 1))
        mean, var, _ = self.predict_device(x, noiseless=noiseless)
        return mean.cpu().numpy()[:, None], var.cpu().numpy()[:, None]

    def predict_device(self, x, noiseless=True, beta=None):
        """Device tensors (mean, var, acq): acq = LCBSC value when beta is given."""
        f, h = self._factor, self._factor['hyper']
        xq = dev.to_device(x).reshape(-1, self.input_dim)
        m = xq.shape[0]
        mean, var = dev.empty((m,)), dev.empty((m,))
        acq = dev.empty((m,)) if beta is not None else None
        _lib.call('elfi_b200_gp_predict_f64', dev.context(), dev.ptr(xq), self.input_dim, m,
                  dev.ptr(f['X']), self.input_dim, f['n'], self.input_dim, dev.ptr(f['W']),
                  f['n_pad'], dev.ptr(f['alpha']), h['kernel_var'], h['lengthscale'],
                  h['bias_var'], 0.0 if noiseless else h['noise_var'],
                  float(beta) if beta is not None else 0.0, dev.ptr(mean), dev.ptr(var),
                  dev.ptr(acq), dev.stream_ptr())
        return mean, var, acq

    def predict_mean(self, x):
        return self.predict(x)[0]

    def predictive_gradients(self, x):
        """Gradients of the GP mean and variance -> ((m, p), (m, p)) (gpy_regression.py:186-223)."""
        x = np.asanyarray(dev.to_host(x), dtype=np.float64).reshape((-1, self.input_dim))
        if self._factor is None:
            return np.zeros((x.shape[0], self.input_dim)), np.zeros((x.shape[0], self.input_dim))
        _, _, gm, gv = self._predict_grad_device(x)
        return gm.cpu().numpy(), gv.cpu().numpy()

    def _predict_grad_device(self, x):
        f, h = self._factor, self._factor['hyper']
        xq = dev.to_device(x).reshape(-1, self.input_dim)
        m, p = xq.shape
        mean, var = dev.empty((m,)), dev.empty((m,))
        gm, gv = dev.empty((m, p)), dev.empty((m, p))
        _lib.call('elfi_b200_gp_predict_grad_f64', dev.context(), dev.ptr(xq), p, m,
                  dev.ptr(f['X']), p, f['n'], p, dev.ptr(f['W']), dev.ptr(f['U']), f['n_pad'],
                  dev.ptr(f['alpha']), h['kernel_var'], h['lengthscale'], h['bias_var'],
                  dev.ptr(mean), dev.ptr(var), dev.ptr(gm), dev.ptr(gv), dev.stream_ptr())
        return mean, var, gm, gv

    def predictive_gradient_mean(self, x):
        return self.predictive_gradients(x)[0]

    def predict_with_gradients(self, x, noiseless=False):
        """mean (m, 1), var (m, 1), grad_mean (m, p), grad_var (m, p) from ONE device call --
        what predict() + predictive_gradients() return together (the posterior / MaxVar
        gradients need all four at the same point)."""
        x = np.asanyarray(dev.to_host(x), dtype=np.float64).reshape((-1, self.input_dim))
        if self._factor is None:
            zeros = np.zeros((x.shape[0], self.input_dim))
            return np.zeros((x.shape[0], 1)), np.ones((x.shape[0], 1)), zeros, zeros.copy()
        mean, var, gm, gv = self._predict_grad_device(x)
        var = var.cpu().numpy()[:, None]
        if not noiseless:
            var = var + self._factor['hyper']['noise_var']
        return mean.cpu().numpy()[:, None], var, gm.cpu().numpy(), gv.cpu().numpy()

    # ---- posterior covariance between points (ExpIntVar) ---------------------------------------
    def whiten(self, x):
        """T (m, n) device tensor with rows W k(x_q, X): cov(a, b) = k(a, b) - T_a . T_b."""
        f, h = self._factor, self._factor['hyper']
        xq = dev.to_device(x).reshape(-1, self.input_dim)
        T = dev.empty((xq.shape[0], f['n']))
        _lib.call('elfi_b200_gp_whiten_f64', dev.context(), dev.ptr(xq), self.input_dim,
                  xq.shape[0], dev.ptr(f['X']), self.input_dim, f['n'], self.input_dim,
                  dev.ptr(f['W']), f['n_pad'], h['kernel_var'], h['lengthscale'], h['bias_var'],
                  dev.ptr(T), f['n'], dev.stream_ptr())
        return xq, T

    def cross_covariance(self, a, b):
        """Noiseless posterior covariance (len(b), len(a)) between two point sets, each given as
        the (points, whitened) pair returned by `whiten` (so a fixed set is whitened once)."""
        (xa, Ta), (xb, Tb) = a, b
        h = self._factor['hyper']
        cov = dev.empty((xb.shape[0], xa.shape[0]))
        _lib.call('elfi_b200_gp_cross_cov_f64', dev.context(), dev.ptr(xa), self.input_dim,
                  xa.shape[0], dev.ptr(Ta), Ta.shape[1], dev.ptr(xb), self.input_dim, xb.shape[0],
                  dev.ptr(Tb), Tb.shape[1], self._factor['n'], self.input_dim, h['kernel_var'],
                  h['lengthscale'], h['bias_var'], dev.ptr(cov), dev.stream_ptr())
        return cov

    # ---- hyper-parameters -------------------------------------------------------------------
    def log_marginal_likelihood(self, hyper=None):
        """-1/2 y^T alpha - sum log L_ii - n/2 log 2 pi for the given (or current) hyper-parameters."""
        f = self._fit(hyper) if hyper is not None else self._factor
        n = f['n']
        diag = torch.diagonal(f['L'])[:n]
        return float(-0.5 * torch.dot(f['y'], f['alpha']) - torch.log(diag).sum()
                     - 0.5 * n * np.log(2 * np.pi))

    def optimize(self):
        """Maximise log marginal likelihood + Gamma log-priors over (kernel_var, lengthscale,
        bias_var, noise_var) in log space.  PARITY UNPINNED w.r.t. GPy's SCG."""
        names = ['kernel_var', 'lengthscale', 'bias_var', 'noise_var']
        # Search box: three decades either side of the initial heuristics.  The Gamma priors of
        # the reference have shape < 1 whenever the heuristic variance is < 1, i.e. an unbounded
        # density at zero; a box tied to the current values would let repeated optimisations walk
        # a variance down to nothing (the GP then explains all evidence as noise).
        anchor = getattr(self, '_hyper_anchor', None) or self._hyper
        centre = np.log([anchor[k] for k in names])
        box = [(c - HYPER_LOG_RANGE, c + HYPER_LOG_RANGE) for c in centre]
        x0 = np.clip(np.log([self._hyper[k] for k in names]), [b[0] for b in box],
                     [b[1] for b in box])

        def objective(logh):
            return -self.log_posterior_hyper(dict(zip(names, np.exp(logh))))
        f0 = objective(x0)
        res = scipy.optimize.minimize(objective, x0, method='L-BFGS-B', bounds=box,
                                      options={'maxiter': self.max_opt_iters})
        if np.isfinite(res.fun) and res.fun <= f0:
            self._hyper = dict(zip(names, np.exp(res.x).tolist()))
        else:
            logger.warning("Numerical error in GP optimization. Stopping optimization")
        self._fit()

    def log_posterior_hyper(self, hyper=None):
        """The quantity `optimize` maximises: log marginal likelihood + Gamma log-priors + the log
        Jacobian of GPy's positivity transform for the priored parameters.  GPy optimises its
        positive parameters through Logexp (x = log(1 + e^u)) and, for a parameter that carries a
        prior, adds log|dx/du| = log(1 - e^-x) to the log-prior (paramz Priorizable.log_prior);
        without that term the reference's Gamma priors with shape < 1 (heuristic variance < 1) are
        unbounded at zero and a full optimisation walks the kernel variance to nothing."""
        h = hyper or self._hyper
        try:
            val = self.log_marginal_likelihood(dict(h))
        except (np.linalg.LinAlgError, _lib.ElfiB200Error):
            return -1e25
        for k, (a, b) in self._priors.items():
            val += ss.gamma.logpdf(h[k], a=a, scale=1.0 / b) + np.log(-np.expm1(-h[k]))
        return val if np.isfinite(val) else -1e25

    def copy(self):
        kopy = copy.copy(self)
        if self._factor is not None:
            kopy._factor = {k: (v.clone() if isinstance(v, torch.Tensor) else copy.copy(v))
                            for k, v in self._factor.items()}
        kopy._hyper = copy.copy(self._hyper)
        return kopy


# ------------------------------------------------------------------------------ acquisition
def _multistart_points(bounds, n, prior, random_state):
    """(n, dim) start points inside the box `bounds`: draws from `prior` clipped to the box, or,
    without a prior, uniform draws taken one coordinate after the other (which is how the
    reference consumes the RandomState, elfi/methods/bo/utils.py:77-88; goldens depend on it)."""
    if prior is None:
        rs = random_state or np.random
        return np.column_stack([rs.uniform(lo, hi, n) for lo, hi in bounds])
    lows, highs = np.asarray(bounds, dtype=float).T
    draws = np.asarray(prior.rvs(n, random_state=random_state)).reshape(n, -1)
    return np.clip(draws, lows, highs)


def _best_of(runs, bounds):
    """The local optimum with the smallest value (first one on ties), clipped to the box."""
    values = np.array([np.ravel(run.fun)[0] for run in runs], dtype=float)
    k = int(np.argmin(values))
    lows, highs = np.asarray(bounds, dtype=float).T
    return np.clip(runs[k].x, lows, highs), values[k]


def minimize(fun, bounds, method='L-BFGS-B', constraints=None, grad=None, prior=None,
             n_start_points=10, maxiter=1000, random_state=None):
    """Multi-start local minimisation with the interface of elfi/methods/bo/utils.py:40-111:
    one SciPy local search per start point, the best end point wins."""
    starts = _multistart_points(bounds, n_start_points, prior, random_state)
    runs = [scipy.optimize.minimize(fun, x0, method=method, jac=grad, bounds=bounds,
                                    constraints=constraints, options=dict(maxiter=maxiter))
            for x0 in starts]
    return _best_of(runs, bounds)


class CostFunction:
    """An acquisition cost: scale * function(x) with its gradient (elfi/methods/bo/utils.py:
    CostFunction).  BOLFIRE adds minus the log prior to LCBSC with it."""

    def __init__(self, function, gradient, scale=1):
        self.function = function
        self.gradient = gradient
        self.scale = scale

    def evaluate(self, x):
        """(n, 1) values at x, (input_dim,) or (n, input_dim)."""
        x = np.atleast_2d(x)
        n, input_dim = x.shape
        return self.scale * np.asarray(self.function(x)).reshape(n, 1)

    def evaluate_gradient(self, x):
        """(n, input_dim) gradients at x."""
        x = np.atleast_2d(x)
        n, input_dim = x.shape
        return self.scale * np.asarray(self.gradient(x)).reshape(n, input_dim)


class _Rendezvous:
    """Meeting point of several local optimisations running in worker threads and the thread
    that owns the device: workers post the point they need and sleep; once every live worker has
    posted, the owner evaluates all points in one batched call and wakes them."""

    def __init__(self, n_workers):
        self.cv = threading.Condition()
        self.live = n_workers
        self.posted = {}
        self.answers = {}
        self.error = None

    def request(self, worker, x):
        with self.cv:
            self.posted[worker] = np.array(x, dtype=float, copy=True)
            self.cv.notify_all()
            while worker not in self.answers and self.error is None:
                self.cv.wait()
            if self.error is not None:
                raise self.error
            return self.answers.pop(worker)

    def retire(self, worker):
        with self.cv:
            self.live -= 1
            self.cv.notify_all()

    def serve(self, batch_fun):
        """Run on the owning thread until all workers have retired."""
        try:
            while True:
                with self.cv:
                    while self.live > 0 and len(self.posted) < self.live:
                        self.cv.wait()
                    if self.live == 0:
                        return
                    workers = sorted(self.posted)
                    X = np.array([self.posted[w] for w in workers])
                    self.posted.clear()
                values, grads = batch_fun(X)
                values = np.ravel(values)
                with self.cv:
                    for k, w in enumerate(workers):
                        self.answers[w] = (float(values[k]), None if grads is None
                                           else np.array(grads[k], dtype=float))
                    self.cv.notify_all()
        except BaseException as exc:     # whatever stops the owner must release the workers
            with self.cv:
                self.error = exc
                self.cv.notify_all()
            raise


def minimize_lockstep(batch_fun, bounds, method='L-BFGS-B', constraints=None, prior=None,
                      n_start_points=10, maxiter=1000, random_state=None, with_grad=True):
    """`minimize` with all starts advancing together: batch_fun(X (k, dim)) -> (values (k,),
    gradients (k, dim) or None) is called once per round with the points the k still-running
    local optimisations are waiting for, i.e. ONE batched GP call on the device instead of one
    per start and point (SURVEY.md section 8f N3).  Start points, local optimiser and selection are
    those of `minimize`, so with the same function values the result is the same.  With
    with_grad=False the optimiser differentiates numerically (batch_fun returns (values, None))."""
    start_points = _multistart_points(bounds, n_start_points, prior, random_state)
    meet = _Rendezvous(n_start_points)
    results = [None] * n_start_points

    def local_search(i):
        try:
            def objective(x):
                value, grad = meet.request(i, x)
                return (value, grad) if with_grad else value
            results[i] = scipy.optimize.minimize(objective, start_points[i, :], method=method,
                                                 jac=True if with_grad else None, bounds=bounds,
                                                 constraints=constraints,
                                                 options={'maxiter': maxiter})
        except BaseException as exc:
            results[i] = exc
        finally:
            meet.retire(i)

    threads = [threading.Thread(target=local_search, args=(i,), daemon=True)
               for i in range(n_start_points)]
    for th in threads:
        th.start()
    try:
        meet.serve(batch_fun)
    finally:
        for th in threads:
            th.join()
    for res in results:
        if isinstance(res, BaseException):
            raise res
    return _best_of(results, bounds)


class AcquisitionBase:
    """elfi/methods/bo/acquisition.py:16-191."""

    def __init__(self, model, prior=None, n_inits=10, max_opt_iters=1000, noise_var=None,
                 exploration_rate=10, seed=None, constraints=None):
        self.model, self.prior, self.constraints = model, prior, constraints
        self.n_inits, self.max_opt_iters = int(n_inits), int(max_opt_iters)
        self.noise_var = self._per_parameter_noise(noise_var)
        self.exploration_rate = exploration_rate
        self.seed = seed or 0
        self.random_state = np.random.RandomState(seed) if seed is not None else np.random

    def _per_parameter_noise(self, noise_var):
        """Acquisition noise variance: None, one non-negative number for all parameters, or
        {parameter name: non-negative number} naming exactly the GP's parameters (returned as a
        list in parameter order).  Anything else is a ValueError."""
        if noise_var is None:
            return None
        names = self.model.parameter_names
        if isinstance(noise_var, dict):
            if set(noise_var) != set(names):
                raise ValueError('The acquisition noise dictionary must name every parameter '
                                 '(and nothing else): {}'.format(names))
            variances = [noise_var[n] for n in names]
        elif isinstance(noise_var, (int, float)):
            variances = [noise_var]
        else:
            raise ValueError('Acquisition noise is a number or a dictionary {parameter name: '
                             'number} of variances')
        for v in variances:
            if not isinstance(v, (int, float)) or v < 0:
                raise ValueError('Acquisition noise variances must be non-negative numbers, '
                                 'got {!r}'.format(v))
        return variances if isinstance(noise_var, dict) else noise_var

    def evaluate(self, x, t=None):
        raise NotImplementedError

    def evaluate_gradient(self, x, t=None):
        raise NotImplementedError

    lockstep = True   # advance the multi-start optimisation with one batched GP call per round

    def evaluate_with_gradient(self, x, t=None):
        """Values (m,) and gradients (m, dim) of a batch of points (default: two calls)."""
        x = np.asanyarray(x, dtype=np.float64).reshape((-1, self.model.input_dim))
        return np.ravel(self.evaluate(x, t)), self.evaluate_gradient(x, t)

    def acquire(self, n, t=None):
        method = 'L-BFGS-B' if self.constraints is None else 'SLSQP'
        if self.lockstep:
            xhat, _ = minimize_lockstep(lambda X: self.evaluate_with_gradient(X, t),
                                        self.model.bounds, method=method,
                                        constraints=self.constraints, prior=self.prior,
                                        n_start_points=self.n_inits, maxiter=self.max_opt_iters,
                                        random_state=self.random_state)
        else:
            xhat, _ = minimize(lambda x: self.evaluate(x, t), self.model.bounds, method=method,
                               constraints=self.constraints,
                               grad=lambda x: self.evaluate_gradient(x, t), prior=self.prior,
                               n_start_points=self.n_inits, maxiter=self.max_opt_iters,
                               random_state=self.random_state)
        x = np.tile(xhat, (n, 1))
        return self._add_noise(x)

    def _add_noise(self, x):
        """Jitter the acquired rows, coordinate by coordinate, with normal noise truncated to
        the GP bounds (acquisition.py:176-191; the coordinate order fixes the RNG stream)."""
        if self.noise_var is None:
            return x
        variances = np.broadcast_to(np.asarray(self.noise_var), (self.model.input_dim,))
        for i, (lo, hi) in enumerate(self.model.bounds):
            sd = np.sqrt(variances[i])
            if sd > 0:
                centre = x[:, i]
                x[:, i] = ss.truncnorm.rvs((lo - centre) / sd, (hi - centre) / sd, loc=centre,
                                           scale=sd, size=len(x), random_state=self.random_state)
        return x


class LCBSC(AcquisitionBase):
    """Lower confidence bound selection criterion (acquisition.py:194-301); the value and its
    gradient are evaluated on the device, fused with the GP prediction."""

    def __init__(self, *args, delta=None, additive_cost=None, **kwargs):
        if delta is not None:             # delta is the reciprocal of the exploration rate
            if not 0 < delta < 1:
                logger.warning('LCBSC: delta = %s is outside (0, 1)', delta)
            kwargs['exploration_rate'] = 1 / delta
        super().__init__(*args, **kwargs)
        self.name, self.label_fn = 'lcbsc', 'Confidence Bound'
        self.additive_cost = additive_cost

    @property
    def delta(self):
        return 1 / self.exploration_rate

    def _beta(self, t):
        t += 1
        d = self.model.input_dim
        return 2 * np.log(t ** (2 * d + 2) * np.pi ** 2 / (3 * self.delta))

    def evaluate(self, x, t=None):
        """(m, 1) host array; use evaluate_device for large grids."""
        value = self.evaluate_device(x, t).cpu().numpy()[:, None]
        if self.additive_cost is not None:
            value += self.additive_cost.evaluate(x)
        return value

    def evaluate_device(self, x, t=None):
        if self.model._factor is None:
            m = np.asarray(dev.to_host(x)).reshape(-1, self.model.input_dim).shape[0]
            return dev.full((m,), -np.sqrt(self._beta(t)))
        return self.model.predict_device(x, noiseless=True, beta=self._beta(t))[2]

    def evaluate_gradient(self, x, t=None):
        return self.evaluate_with_gradient(x, t, want_value=False)[1]

    def evaluate_with_gradient(self, x, t=None, want_value=True):
        """LCBSC values (m,) and gradients (m, dim) from one GP launch + one epilogue launch."""
        x = np.asanyarray(x, dtype=np.float64).reshape((-1, self.model.input_dim))
        if self.model._factor is None:
            return np.full(len(x), -np.sqrt(self._beta(t))), np.zeros_like(x)
        mean, var, gm, gv = self.model._predict_grad_device(x)
        m, p = gm.shape
        acq = dev.empty((m,)) if want_value else None
        gacq = dev.empty((m, p))
        _lib.call('elfi_b200_lcbsc_f64', dev.context(), dev.ptr(mean), dev.ptr(var), dev.ptr(gm),
                  dev.ptr(gv), m, p, float(self._beta(t)), dev.ptr(acq), dev.ptr(gacq),
                  dev.stream_ptr())
        value = acq.cpu().numpy() if want_value else None
        grad = gacq.cpu().numpy()
        if self.additive_cost is not None:
            if want_value:
                value = value + np.ravel(self.additive_cost.evaluate(x))
            grad += self.additive_cost.evaluate_gradient(x)
        return value, grad


class MaxVar(AcquisitionBase):
    """Acquire where the variance of the unnormalised approximate posterior
    prior(theta)^2 * Var[Phi((eps - f(theta)) / sigma_n)] is largest (Jarvenpaa et al. 2019;
    elfi/methods/bo/acquisition.py:304-469).  eps is the `quantile_eps` quantile of the evidence
    discrepancies.  The GP moments and their gradients at a point come from one device call."""

    def __init__(self, model, prior, quantile_eps=.01, **opts):
        super().__init__(model, prior=prior, **opts)
        self.name = 'max_var'
        self.label_fn = 'Variance of the Unnormalised Approximate Posterior'
        self.quantile_eps = quantile_eps
        self.eps = .1   # until the first acquire(): the GP is not fitted yet

    def _update_eps(self):
        self.eps = np.percentile(self.model.Y, self.quantile_eps * 100)

    def acquire(self, n, t=None):
        logger.debug('Acquiring the next batch of %d values', n)
        self._update_eps()
        if self.lockstep:
            theta_max, _ = minimize_lockstep(
                lambda X: (-np.ravel(self.evaluate(X)), -self.evaluate_gradient(X)),
                self.model.bounds, prior=self.prior, n_start_points=self.n_inits,
                maxiter=self.max_opt_iters, random_state=self.random_state)
        else:
            theta_max, _ = minimize(lambda theta: -self.evaluate(theta), self.model.bounds,
                                    grad=lambda theta: -self.evaluate_gradient(theta),
                                    prior=self.prior, n_start_points=self.n_inits,
                                    maxiter=self.max_opt_iters, random_state=self.random_state)
        return np.tile(theta_max, (n, 1))   # the same location for the whole batch

    def _gp(self, theta):
        theta = np.asanyarray(theta, dtype=float).reshape((-1, self.model.input_dim))
        if hasattr(self.model, 'predict_with_gradients'):
            return (theta,) + tuple(self.model.predict_with_gradients(theta, noiseless=True))
        return (theta,) + tuple(self.model.predict(theta, noiseless=True)) + \
            tuple(self.model.predictive_gradients(theta))

    def evaluate(self, theta_new, t=None):
        """Var[p_a] = Phi_skew(eps) - Phi(eps)^2: a skew-normal cdf stands in for Owen's T."""
        theta, mean, var = self._gp(theta_new)[:3]
        sigma2_n = self.model.noise
        skew = np.sqrt(sigma2_n) / np.sqrt(sigma2_n + 2. * var)
        scale = np.sqrt(sigma2_n + var)
        var_p_a = ss.skewnorm.cdf(self.eps, skew, loc=mean, scale=scale) \
            - ss.norm.cdf(self.eps, loc=mean, scale=scale) ** 2
        prior = self.prior.pdf(theta_new).ravel()[:, np.newaxis]
        return prior ** 2 * var_p_a

    def evaluate_gradient(self, theta_new, t=None):
        theta, mean, var, grad_mean, grad_var = self._gp(theta_new)
        sigma2_n = self.model.noise
        phi = ss.norm.cdf
        scale = np.sqrt(sigma2_n + var)
        a = (self.eps - mean) / scale
        b = np.sqrt(sigma2_n) / np.sqrt(sigma2_n + 2 * var)
        grad_a = (-1. / scale) * grad_mean \
            - ((self.eps - mean) / (2. * (sigma2_n + var) ** 1.5)) * grad_var
        grad_b = (-np.sqrt(sigma2_n) / (sigma2_n + 2 * var) ** 1.5) * grad_var
        phi_a = phi(a)
        gauss_a = np.exp(-.5 * a ** 2)
        int_1 = phi_a - phi_a ** 2
        int_2 = phi(self.eps, loc=mean, scale=scale) \
            - ss.skewnorm.cdf(self.eps, b, loc=mean, scale=scale)
        grad_int_1 = (1. - 2 * phi_a) * (gauss_a / np.sqrt(2. * np.pi)) * grad_a
        grad_int_2 = (1. / np.pi) * (
            (np.exp(-.5 * a ** 2 * (1. + b ** 2)) / (1. + b ** 2)) * grad_b
            + np.sqrt(np.pi / 2.) * gauss_a * (1. - 2. * phi(a * b)) * grad_a)
        prior = self.prior.pdf(theta_new).ravel()[:, np.newaxis]
        grad_prior = prior * self.prior.gradient_logpdf(theta_new)   # f' = (log f)' f
        return 2. * prior * (int_1 - int_2) * grad_prior + prior ** 2 * (grad_int_1 - grad_int_2)


class RandMaxVar(MaxVar):
    """Sample the next point from the MaxVar surface, treated as an unnormalised density, with a
    short MCMC chain (acquisition.py:472-626)."""

    def __init__(self, model, prior, quantile_eps=.01, sampler='nuts', n_samples=50, warmup=None,
                 limit_faulty_init=1000, init_from_prior=False, sigma_proposals=None, **opts):
        super().__init__(model, prior, quantile_eps, **opts)
        self.name = 'rand_max_var'
        self.name_sampler = sampler
        self._n_samples = n_samples
        self._warmup = warmup or n_samples // 2
        self._limit_faulty_init = limit_faulty_init
        self._init_from_prior = init_from_prior
        if self.name_sampler == 'metropolis':
            self._sigma_proposals = resolve_sigmas(self.model.parameter_names, sigma_proposals,
                                                   self.model.bounds)

    def _initial_point(self):
        bounds = self.model.bounds
        if self._init_from_prior:
            theta = self.prior.rvs(random_state=self.random_state)
            return np.array([np.clip(theta[i], lo, hi) for i, (lo, hi) in enumerate(bounds)])
        return np.array([self.random_state.uniform(lo, hi) for lo, hi in bounds])

    def acquire(self, n, t=None):
        if n > self._n_samples:
            raise ValueError(("The number of acquisitions ({0}) has to be lower than the number "
                              "of the samples ({1}).").format(n, self._n_samples - self._warmup))
        logger.debug('Acquiring the next batch of %d values', n)
        self._update_eps()

        def logpdf(theta):
            value = float(np.ravel(self.evaluate(theta))[0])
            return -np.inf if value == 0 else np.log(value)

        def gradient_logpdf(theta):
            value = float(np.ravel(self.evaluate(theta))[0])
            return -np.inf if value == 0 else (self.evaluate_gradient(theta) / value).ravel()

        for _ in range(self._limit_faulty_init):
            theta_init = self._initial_point()
            if not np.isinf(logpdf(theta_init)):
                break
        else:
            raise SystemExit("Unable to find a suitable initial point.")
        if self.name_sampler == 'metropolis':
            samples = mcmc.metropolis(self._n_samples, theta_init, logpdf,
                                      sigma_proposals=self._sigma_proposals, seed=self.seed)
        elif self.name_sampler == 'nuts':
            samples = mcmc.nuts(self._n_samples, theta_init, logpdf, gradient_logpdf,
                                seed=self.seed)
        else:
            raise ValueError("Incompatible sampler. Please check the options in the documentation.")
        if n > 1:
            return self.random_state.permutation(samples[self._warmup:])[:n]
        return samples[-1:]


class ExpIntVar(MaxVar):
    """Expected integrated variance (Jarvenpaa et al. 2019; acquisition.py:629-821): choose the
    point whose simulation is expected to reduce the variance of the unnormalised posterior most,
    integrated over a grid of the parameter space or over importance samples drawn from the MaxVar
    surface.  The posterior covariance between the integration points and a candidate is
    k(i, c) - (W k_i) . (W k_c) on the device, with the integration points whitened once per
    acquisition (the reference re-factorises Ky in every evaluation)."""

    def __init__(self, model, prior, quantile_eps=.01, integration='grid', d_grid=.2,
                 n_samples_imp=100, iter_imp=2, sampler='nuts', n_samples=2000,
                 sigma_proposals=None, **opts):
        super().__init__(model, prior, quantile_eps, **opts)
        self.name = 'exp_int_var'
        self.label_fn = 'Expected Loss'
        self._integration = integration
        self._n_samples_imp = n_samples_imp
        self._iter_imp = iter_imp
        if self._integration == 'importance':
            self.density_is = RandMaxVar(model=self.model, prior=self.prior, n_inits=self.n_inits,
                                         seed=self.seed, quantile_eps=self.quantile_eps,
                                         sampler=sampler, n_samples=n_samples,
                                         sigma_proposals=sigma_proposals)
        elif self._integration == 'grid':
            axes = [slice(b[0], b[1], d_grid) for b in self.model.bounds]
            self.points_int = np.mgrid[axes].reshape(len(self.model.bounds), -1).T

    def _prepare(self, t):
        """Everything of the expected loss that does not depend on the candidate point."""
        gp = self.model
        self.sigma2_n = gp.noise
        self._update_eps()
        resample = self._integration == 'importance' and t % self._iter_imp == 0
        if resample:
            self.points_int = self.density_is.acquire(self._n_samples_imp)
        self.mean_int, self.var_int = gp.predict(self.points_int, noiseless=True)
        self.priors_int = (self.prior.pdf(self.points_int) ** 2)[np.newaxis, :]
        if resample:
            omegas = (1 / MaxVar.evaluate(self, self.points_int)).T
            self.omegas_int = omegas / np.sum(omegas, axis=1)[:, np.newaxis]
        elif self._integration == 'grid':
            self.omegas_int = np.full(len(self.points_int), 1 / len(self.points_int))
        self._whitened_int = gp.whiten(self.points_int)
        self.phi_int = ss.norm.cdf(self.eps, loc=self.mean_int.T,
                                   scale=np.sqrt(self.sigma2_n + self.var_int.T))

    def acquire(self, n, t):
        logger.debug('Acquiring the next batch of %d values', n)
        self._prepare(t)
        if self.lockstep:
            theta_min, _ = minimize_lockstep(lambda X: (self.evaluate(X), None), self.model.bounds,
                                             prior=self.prior, n_start_points=self.n_inits,
                                             maxiter=self.max_opt_iters,
                                             random_state=self.random_state, with_grad=False)
        else:
            theta_min, _ = minimize(self.evaluate, self.model.bounds, grad=None, prior=self.prior,
                                    n_start_points=self.n_inits, maxiter=self.max_opt_iters,
                                    random_state=self.random_state)
        return np.tile(theta_min, (n, 1))

    def evaluate(self, theta_new, t=None):
        """The candidate-dependent term of the expected loss (to be minimised)."""
        gp = self.model
        theta_new = np.asanyarray(theta_new, dtype=float).reshape((-1, gp.input_dim))
        _, var_new = gp.predict(theta_new, noiseless=True)
        cov_int = dev.to_host(gp.cross_covariance(self._whitened_int, gp.whiten(theta_new)))
        delta_var_int = cov_int ** 2 / (self.sigma2_n + var_new)
        spread = self.sigma2_n + self.var_int.T
        a = np.sqrt((spread - delta_var_int) / (spread + delta_var_int))
        phi_skew = ss.skewnorm.cdf(self.eps, a, loc=self.mean_int.T, scale=np.sqrt(spread))
        w = (self.phi_int - phi_skew) / 2
        loss = 2 * np.sum(self.omegas_int * self.priors_int * w, axis=1)
        return np.where(self.prior.pdf(theta_new) == 0, np.finfo(float).max, loss)


class UniformAcquisition(AcquisitionBase):
    """Uniform draws inside the GP bounds (acquisition.py:824-845)."""

    def acquire(self, n, t=None):
        bounds = np.stack(self.model.bounds)
        return ss.uniform(bounds[:, 0], bounds[:, 1] - bounds[:, 0]).rvs(
            size=(n, self.model.input_dim), random_state=self.random_state)


# ------------------------------------------------------------------------------------ BO loop
def ceil_to_batch_size(num, batch_size):
    return int(batch_size * ceil(num / batch_size))


class BayesianOptimization(ParameterInference):
    """Sequential Bayesian optimisation of a model output (the discrepancy) over the parameters:
    a GP surrogate of output against parameters, updated with every finished batch, and an
    acquisition rule that proposes where to simulate next.  Interface of
    elfi/methods/inference/bolfi.py:26-292.

    Evidence bookkeeping: the first `n_initial_evidence` points come from the prior (or are
    handed in precomputed); from then on batch b uses acquisition round
    ``(b * batch_size - n_initial_to_simulate) // acq_batch_size`` and the GP hyper-parameters are
    re-optimised whenever `update_interval` new points have arrived since the last time."""

    def __init__(self, model, target_name=None, bounds=None, initial_evidence=None,
                 update_interval=10, target_model=None, acquisition_method=None, acq_noise_var=0,
                 exploration_rate=10, batch_size=1, batches_per_acquisition=None, async_acq=False,
                 **kwargs):
        model, target_name = self._resolve_model(model, target_name)
        super().__init__(model, [target_name] + model.parameter_names, batch_size=batch_size,
                         **kwargs)
        self.target_name = target_name
        self.target_model = target_model or GPyRegression(self.model.parameter_names,
                                                          bounds=bounds)
        self.update_interval, self.async_acq = update_interval, async_acq
        self.batches_per_acquisition = batches_per_acquisition or self.max_parallel_batches
        self.n_initial_evidence, given = self._initial_evidence_plan(initial_evidence)
        self.n_precomputed_evidence = 0
        if given is not None:
            theta = np.column_stack([given[n] for n in self.target_model.parameter_names])
            self.target_model.update(theta, given[target_name])
            self.n_precomputed_evidence = len(theta)
        if acquisition_method is None:
            acquisition_method = LCBSC(
                self.target_model, noise_var=acq_noise_var, exploration_rate=exploration_rate,
                seed=self.seed,
                prior=ModelPrior(self.model, parameter_names=self.target_model.parameter_names))
        self.acquisition_method = acquisition_method
        self.state.update(n_evidence=self.n_precomputed_evidence,
                          last_GP_update=self.n_initial_evidence, acquisition=[])

    def _initial_evidence_plan(self, initial_evidence):
        """(number of evidence points that precede the first acquisition, precomputed outputs or
        None).  None asks for max(10, 2^dim + 1) points, a number for that many -- both rounded
        up to whole batches since they are simulated; a dict of outputs is used as it is."""
        if initial_evidence is None:
            count = max(10, 2 ** self.target_model.input_dim + 1)
        elif np.isscalar(initial_evidence):
            count = int(initial_evidence)
            if count < 0:
                raise ValueError('The number of initial evidence points cannot be negative '
                                 '(got {})'.format(initial_evidence))
        else:
            return len(initial_evidence[self.target_name]), initial_evidence
        return ceil_to_batch_size(count, self.batch_size), None

    @property
    def n_evidence(self):
        return self.state.get('n_evidence', 0)

    @property
    def acq_batch_size(self):
        """Points requested from the acquisition rule at a time."""
        return self.batches_per_acquisition * self.batch_size

    def set_objective(self, n_evidence=None):
        """Run until the surrogate holds `n_evidence` points (precomputed ones count)."""
        if n_evidence is None:
            n_evidence = self.objective.get('n_evidence', self.n_evidence)
        self.objective.update(n_evidence=n_evidence,
                              n_sim=n_evidence - self.n_precomputed_evidence)

    def _as_parameter_dict(self, rows):
        names = self.target_model.parameter_names
        rows = np.asarray(rows).reshape((-1, len(names)))
        return {name: rows[:, i] for i, name in enumerate(names)}

    def extract_result(self):
        """The minimiser of the surrogate mean (global search inside the bounds, then polish)
        and all evidence gathered so far."""
        gp = self.target_model
        found = scipy.optimize.differential_evolution(
            lambda x: gp.predict_mean(x).ravel(), gp.bounds, maxiter=1000, polish=True,
            init='latinhypercube', seed=self.seed)
        outputs = self._as_parameter_dict(gp.X)
        outputs[self.target_name] = gp.Y
        return OptimizationResult(x_min=self._as_parameter_dict(found.x), outputs=outputs,
                                  **self._extract_result_kwargs())

    def update(self, batch, batch_index):
        """A finished batch becomes evidence of the surrogate."""
        super().update(batch, batch_index)
        self.state['n_evidence'] += self.batch_size
        gp = self.target_model
        theta = np.column_stack([np.asarray(dev.to_host(batch[n])) for n in gp.parameter_names])
        reoptimise = self._should_optimize()
        gp.update(theta, dev.to_host(batch[self.target_name]), reoptimise)
        if reoptimise:
            self.state['last_GP_update'] = gp.n_evidence

    def prepare_new_batch(self, batch_index):
        """Parameter values for the next batch: None while the initial evidence is being drawn
        from the prior, afterwards the next `batch_size` rows of the pending acquisition (a new
        one is requested when none are left)."""
        t = self._get_acquisition_index(batch_index)
        if t < 0:
            return None
        pending = self.state['acquisition']
        if len(pending) == 0:
            pending = self.acquisition_method.acquire(self.acq_batch_size, t=t)
        self.state['acquisition'] = pending[self.batch_size:]
        return self._as_parameter_dict(pending[:self.batch_size])

    def _get_acquisition_index(self, batch_index):
        to_simulate_first = self.n_initial_evidence - self.n_precomputed_evidence
        return (batch_index * self.batch_size - to_simulate_first) // self.acq_batch_size

    def _should_optimize(self):
        """Re-optimise the hyper-parameters with this update?  Once the initial evidence is
        complete, every `update_interval` points."""
        after = self.target_model.n_evidence + self.batch_size
        due = self.state['last_GP_update'] + self.update_interval
        return after >= max(self.n_initial_evidence, due)


class BolfiPosterior:
    """Unnormalised BOLFI posterior  prior(x) * Phi((h - mu(x)) / sigma(x))  with the GP mean and
    the noisy GP standard deviation (elfi/methods/posteriors.py:21-189).  Zero outside the GP
    bounds.  logpdf and gradient_logpdf at the same point share one device call."""

    def __init__(self, model, threshold=None, prior=None, n_inits=10, max_opt_iters=1000, seed=0):
        self.model = model
        self.threshold = threshold
        self.prior = prior
        self.dim = self.model.input_dim
        self.random_state = np.random.RandomState(seed)
        self.n_inits = n_inits
        self.max_opt_iters = max_opt_iters
        self._memo = (None, None)
        if self.threshold is None:   # minimum of the GP mean (posteriors.py:62-73)
            _, minval = minimize(self.model.predict_mean, self.model.bounds,
                                 grad=self.model.predictive_gradient_mean, prior=self.prior,
                                 n_start_points=self.n_inits, maxiter=self.max_opt_iters,
                                 random_state=self.random_state)
            self.threshold = minval
            logger.info("Using optimized minimum value (%.4f) of the GP discrepancy mean "
                        "function as a threshold" % (self.threshold))

    def rvs(self, size=None, random_state=None):
        raise NotImplementedError('Currently not implemented. Please use a sampler to '
                                  'sample from the posterior.')

    # ---- GP moments at the points inside the bounds -------------------------------------------
    def _rows(self, x):
        x = np.asanyarray(x)
        scalar = x.ndim == 0 or (x.ndim == 1 and self.dim > 1)
        return x.reshape((-1, self.dim)), scalar

    def _within_bounds(self, x):
        x = x.reshape((-1, self.dim))
        lo = np.array([b[0] for b in self.model.bounds])
        hi = np.array([b[1] for b in self.model.bounds])
        return np.all((x >= lo) & (x <= hi), axis=1)

    def _moments(self, x):
        key = x.tobytes()
        if self._memo[0] != key:
            if hasattr(self.model, 'predict_with_gradients'):
                out = self.model.predict_with_gradients(x)
            else:
                out = self.model.predict(x) + self.model.predictive_gradients(x)
            self._memo = (key, out)
        return self._memo[1]

    def _unnormalized_loglikelihood(self, x):
        x, scalar = self._rows(x)
        logpdf = np.full(len(x), -np.inf)
        inside = self._within_bounds(x)
        if inside.any():
            mean, var = self._moments(np.ascontiguousarray(x[inside]))[:2]
            logpdf[inside] = ss.norm.logcdf(self.threshold, mean, np.sqrt(var)).squeeze()
        return logpdf[0] if scalar else logpdf

    def _gradient_unnormalized_loglikelihood(self, x):
        x, scalar = self._rows(x)
        grad = np.zeros_like(x, dtype=float)
        inside = self._within_bounds(x)
        if inside.any():
            mean, var, grad_mean, grad_var = self._moments(np.ascontiguousarray(x[inside]))
            std = np.sqrt(var)
            z = (self.threshold - mean) / std
            dz = (-grad_mean * std - (self.threshold - mean) * 0.5 * grad_var / std) / var
            grad[inside, :] = dz * ss.norm.pdf(z) / ss.norm.cdf(z)
        return grad[0] if scalar else grad

    def logpdf(self, x):
        return self._unnormalized_loglikelihood(x) + self.prior.logpdf(x)

    def pdf(self, x):
        return np.exp(self.logpdf(x))

    def gradient_logpdf(self, x):
        return self._gradient_unnormalized_loglikelihood(x) + self.prior.gradient_logpdf(x)

    def _unnormalized_likelihood(self, x):
        return np.exp(self._unnormalized_loglikelihood(x))

    def logpdf_and_gradient(self, x, with_grad=True):
        """logpdf (k,) and gradient_logpdf (k, dim) of k points from one device call: the batched
        evaluator of mcmc.run_lockstep (all chains of BOLFI.sample advance together)."""
        x = np.ascontiguousarray(np.asanyarray(x, dtype=float).reshape((-1, self.dim)))
        logpdf = np.atleast_1d(self.logpdf(x))
        grad = np.atleast_2d(self.gradient_logpdf(x)) if with_grad else None   # moments memoised
        return logpdf, grad


class BOLFI(BayesianOptimization):
    """Bayesian optimisation for likelihood-free inference (bolfi.py:400-462)."""

    def fit(self, n_evidence, threshold=None, bar=True):
        if n_evidence is None:
            raise ValueError('You must specify the number of evidence (n_evidence) for the fitting')
        self.infer(n_evidence, bar=bar)
        return self.extract_posterior(threshold)

    def extract_posterior(self, threshold=None):
        if self.state['n_evidence'] == 0:
            raise ValueError('Model is not fitted yet, please see the `fit` method.')
        prior = ModelPrior(self.model, parameter_names=self.target_model.parameter_names)
        return BolfiPosterior(self.target_model, threshold=threshold, prior=prior)

    def sample(self, n_samples, warmup=None, n_chains=4, threshold=None, initials=None,
               algorithm='nuts', sigma_proposals=None, n_evidence=None, **kwargs):
        """Draw from the BOLFI posterior with `n_chains` NUTS (default) or Metropolis chains of
        `n_samples` iterations each, warm-up included (bolfi.py:464-598).  Chains start from the
        evidence points with the smallest discrepancies unless `initials` (n_chains, n_params) is
        given; chain i is seeded with get_sub_seed(seed, i).  `lockstep=False` runs the chains one
        after the other like the reference's client does; the draws are the same either way (a
        chain owns its RandomState).  Returns a BolfiSample."""
        if self.state['n_batches'] == 0:
            self.fit(n_evidence)
        if algorithm not in ['nuts', 'metropolis']:
            raise ValueError("Unknown posterior sampler.")
        posterior = self.extract_posterior(threshold)
        warmup = warmup or n_samples // 2
        if initials is not None:
            if np.asarray(initials).shape != (n_chains, self.target_model.input_dim):
                raise ValueError("The shape of initials must be (n_chains, n_params).")
            initials = np.asarray(initials, dtype=float)
        else:
            initials = np.asarray(self.target_model.X[np.argsort(self.target_model.Y[:, 0])])
        if algorithm == 'metropolis':
            sigma_proposals = resolve_sigmas(self.target_model.parameter_names, sigma_proposals,
                                             self.target_model.bounds)
        lockstep = kwargs.pop('lockstep', True)
        self.target_model.is_sampling = True
        coroutines = []
        start = 0
        for chain in range(n_chains):
            seed = get_sub_seed(self.seed, chain)
            while np.isinf(posterior.logpdf(initials[start])):   # skip zero-density starts
                start += 1
                if start == len(initials):
                    raise ValueError(
                        "BOLFI.sample: Cannot find enough acceptable initialization points!")
            if algorithm == 'nuts':
                coroutines.append(mcmc.nuts_chain(n_samples, initials[start], n_adapt=warmup,
                                                  seed=seed, **kwargs))
            else:
                coroutines.append(mcmc.metropolis_chain(n_samples, initials[start],
                                                        sigma_proposals, warmup, seed=seed,
                                                        **kwargs))
            start += 1
        if lockstep:
            # all chains advance together: every round of pending density / gradient requests is
            # answered by one batched GP call instead of one call per chain and point
            chains = mcmc.run_lockstep(coroutines, posterior.logpdf_and_gradient)
        else:
            chains = [mcmc._run_single(c, posterior.logpdf, posterior.gradient_logpdf)
                      for c in coroutines]
        chains = np.asarray(chains)
        self.target_model.is_sampling = False
        logger.info("{} chains of {} iterations acquired. Effective sample size and Rhat for each "
                    "parameter:".format(n_chains, n_samples))
        for i, name in enumerate(self.target_model.parameter_names):
            logger.info("{} {} {}".format(name, mcmc.eff_sample_size(chains[:, :, i]),
                                          mcmc.gelman_rubin_statistic(chains[:, :, i])))
        return BolfiSample(method_name='BOLFI', chains=chains,
                           parameter_names=self.target_model.parameter_names, warmup=warmup,
                           threshold=float(posterior.threshold), n_sim=self.state['n_evidence'],
                           seed=self.seed)
