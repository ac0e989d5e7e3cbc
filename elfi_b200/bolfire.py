"""BOLFIRE (Thomas et al., Likelihood-free inference by ratio estimation) with the classifier
fitted on the device.

Host control flow follows the reference (paths relative to elfi-dev/elfi):
  BOLFIRE                                   elfi/methods/inference/bolfire.py
  ModelBased (rounds of n_training_data)    elfi/methods/inference/parameter_inference.py
                                            (model_based.py, shared with BSL)
  BOLFIREPosterior                          elfi/methods/posteriors.py
  LogisticRegression                        elfi/methods/classifier.py (classifier.py)
Each round simulates n_training_data times at one parameter: a prior draw for the first
n_initial_evidence rounds, the LCBSC acquisition (minus the log prior as an additive cost) after
that.  The round's features and the marginal data share one (n + m, d) device buffer, the
marginal rows written once; the device classifier fits it, predicts the log ratio at the
observed features, and the host reads the log ratio together with the classifier's attributes in
one copy.  The GP surrogate of minus the log ratio is updated with it.

A host model works the same way (its features are uploaded once per batch).  A user Classifier
gets NumPy (X, y) and runs on the host.
"""
import logging
from collections import OrderedDict

import numpy as np
import torch

from . import device as dev
from . import mcmc
from . import ops
from .bo import LCBSC, AcquisitionBase, CostFunction, GPyRegression, minimize
from .classifier import Classifier, LogisticRegression
from .model import get_sub_seed
from .model_based import ModelBased, feature_columns
from .results import BOLFIRESample
from .samplers import ModelPrior, resolve_sigmas

logger = logging.getLogger(__name__)

__all__ = ['BOLFIRE', 'BOLFIREPosterior']


class BOLFIREPosterior:
    """Unnormalised BOLFIRE posterior: log prior(x) minus the GP mean of minus the log ratio
    (elfi/methods/posteriors.py BOLFIREPosterior)."""

    def __init__(self, parameter_names, model, prior, classifier_attributes):
        self._parameter_names = parameter_names
        self._model = model
        self._prior = prior
        self._classifier_attributes = classifier_attributes
        self.dim = model.input_dim

    @property
    def classifier_attributes(self):
        return self._classifier_attributes

    @property
    def surrogate_model_attributes(self):
        """The GP's hyper-parameters in GPy's param_array order (RBF variance, RBF lengthscale,
        bias variance, noise variance) and its evidence."""
        h = self._model.hyperparameters
        return {'parameters': [h['kernel_var'], h['lengthscale'], h['bias_var'], h['noise_var']],
                'X': self._model.X.tolist(), 'Y': self._model.Y.tolist()}

    def pdf(self, x):
        return np.exp(self.logpdf(x))

    def logpdf(self, x):
        """(n, 1) unnormalised log posterior."""
        return np.asarray(self._prior.logpdf(x)).reshape(-1, 1) - self._model.predict_mean(x)

    def gradient_pdf(self, x):
        return np.exp(self.logpdf(x)) * self.gradient_logpdf(x)

    def gradient_logpdf(self, x):
        """(n, dim) gradient of the unnormalised log posterior."""
        grad = np.asarray(self._prior.gradient_logpdf(x)).reshape(-1, self.dim)
        return grad - self._model.predictive_gradient_mean(x)

    def logpdf_and_gradient(self, x, with_grad=True):
        """logpdf (k,) and gradient_logpdf (k, dim) of k points: the batched evaluator of
        mcmc.run_lockstep (all chains of BOLFIRE.sample advance together)."""
        x = np.ascontiguousarray(np.asanyarray(x, dtype=float).reshape((-1, self.dim)))
        logpdf = np.ravel(self.logpdf(x))
        grad = self.gradient_logpdf(x) if with_grad else None
        return logpdf, grad

    def compute_map_estimates(self, n_opt_inits=10, max_opt_iters=1000):
        """The maximiser of the unnormalised posterior inside the GP bounds, per parameter."""
        x, _ = minimize(fun=lambda x: -float(np.ravel(self.logpdf(x))[0]),
                        bounds=self._model.bounds,
                        grad=lambda x: -np.ravel(self.gradient_logpdf(x)),
                        prior=self._prior, n_start_points=n_opt_inits, maxiter=max_opt_iters)
        return OrderedDict((p, x[i]) for i, p in enumerate(self._model.parameter_names))


class BOLFIRE(ModelBased):
    """Bayesian optimisation and classification in likelihood-free inference.  Runs on this rank
    only."""

    D_MAX = ops.LOGREG_D_MAX

    def __init__(self, model, n_training_data, feature_names=None, marginal=None,
                 seed_marginal=None, classifier=None, bounds=None, n_initial_evidence=0,
                 acq_noise_var=0, exploration_rate=10, update_interval=1, target_model=None,
                 acquisition_method=None, **kwargs):
        super().__init__(model, n_training_data, feature_names=feature_names, **kwargs)
        self._random_state = np.random.RandomState(self.seed)
        self.marginal = self._resolve_marginal(marginal, seed_marginal)
        self.classifier = self._resolve_classifier(classifier)
        self.bounds = bounds
        self.acq_noise_var = acq_noise_var
        self.exploration_rate = exploration_rate
        self.update_interval = update_interval
        self.target_model = self._resolve_target_model(target_model)
        self.prior = ModelPrior(self.model, parameter_names=self.parameter_names)
        self.n_initial_evidence = self._resolve_n_initial_evidence(n_initial_evidence)
        self.acquisition_method = self._resolve_acquisition_method(acquisition_method)
        self.state['n_evidence'] = 0
        self.state['last_GP_update'] = self.n_initial_evidence
        self.classifier_attributes = []
        self._setup_training_buffer()
        self._init_round()

    @property
    def parameter_names(self):
        return self.target_model.parameter_names

    @property
    def n_evidence(self):
        return self.state['n_evidence']

    @property
    def current_params(self):
        return self._current_params

    @current_params.setter
    def current_params(self, params):
        self._current_params = params

    def extract_result(self):
        return BOLFIREPosterior(self.parameter_names, self.target_model, self.prior,
                                self.classifier_attributes)

    # ---- resolvers --------------------------------------------------------------------------
    def _resolve_marginal(self, marginal, seed_marginal=None):
        """The marginal data: generated (and kept on the device) when not given, else a 2-d
        array of d columns."""
        if marginal is None:
            marginal = self._generate_marginal(seed_marginal)
            logger.info('New marginal data ({} x {}) are generated.'.format(*marginal.shape))
            return marginal
        if (isinstance(marginal, np.ndarray) or dev.is_device_array(marginal)) and \
                len(marginal.shape) == 2:
            if marginal.shape[1] != self.observed.size:
                raise ValueError('marginal has {} columns, the features {}'.format(
                    marginal.shape[1], self.observed.size))
            return marginal
        raise TypeError('marginal must be 2d numpy array.')

    def _generate_marginal(self, seed_marginal=None):
        batch = self.model.generate(self.n_sim_round, outputs=self.feature_names,
                                    seed=seed_marginal)
        blocks = feature_columns(batch, self.feature_names, self.n_sim_round)
        return blocks[0].contiguous() if len(blocks) == 1 else torch.cat(blocks, dim=1)

    def _resolve_classifier(self, classifier):
        if classifier is None:
            return LogisticRegression()
        if isinstance(classifier, Classifier):
            return classifier
        raise ValueError('classifier must be an instance of Classifier.')

    def _resolve_n_initial_evidence(self, n_initial_evidence):
        if isinstance(n_initial_evidence, int) and n_initial_evidence >= 0:
            return n_initial_evidence
        raise ValueError('n_initial_evidence must be a non-negative integer.')

    def _resolve_target_model(self, target_model):
        if target_model is None:
            return GPyRegression(self.model.parameter_names, self.bounds)
        if isinstance(target_model, GPyRegression):
            return target_model
        raise TypeError('target_model must be an instance of GPyRegression.')

    def _resolve_acquisition_method(self, acquisition_method):
        if acquisition_method is None:
            cost = CostFunction(self.prior.logpdf, self.prior.gradient_logpdf, scale=-1)
            return LCBSC(model=self.target_model, prior=self.prior, noise_var=self.acq_noise_var,
                         exploration_rate=self.exploration_rate, seed=self.seed,
                         additive_cost=cost)
        if isinstance(acquisition_method, AcquisitionBase):
            return acquisition_method
        raise TypeError('acquisition_method must be an instance of AcquisitionBase.')

    # ---- rounds -----------------------------------------------------------------------------
    def _setup_training_buffer(self):
        """One (n + m, d) device buffer: the round's simulations in the first n rows (written by
        _merge_batch through the view `_sim`), the m marginal rows after them, written once;
        labels +1 then -1, on the device.  With the device classifier, `_round_out` receives its
        fit block and the log ratio, for one read per round."""
        n, d = self.n_sim_round, self.observed.size
        m = int(self.marginal.shape[0])
        self._train = dev.empty((n + m, d))
        self._train[n:] = dev.to_device(self.marginal).reshape(m, d)
        self._sim = self._train[:n]
        self._labels_host = np.concatenate([np.ones(n), -np.ones(m)])
        self._device_clf = isinstance(self.classifier, LogisticRegression)
        if self._device_clf:
            self._labels = dev.to_device(self._labels_host)
            self._obs_dev = dev.to_device(self.observed.reshape(1, -1))
            self._round_out = dev.empty((ops.logreg_block_size(d) + 1,))
        self._marginal_host = None

    def _init_round(self):
        super()._init_round()
        if self.n_evidence < self.n_initial_evidence:
            self.current_params = self.prior.rvs(1, random_state=self._random_state)
        else:
            t = self.n_evidence - self.n_initial_evidence
            self.current_params = self.acquisition_method.acquire(1, t)

    def predict_log_ratio(self, X, y, X_obs):
        """Fit the classifier to (X, y) and return its log ratio at X_obs."""
        self.classifier.fit(X, y)
        return self.classifier.predict_log_likelihood_ratio(X_obs)

    def _log_ratio(self):
        """The round's log ratio at the observed features, (1,)."""
        if self._device_clf:
            clf, out = self.classifier, self._round_out
            blk = ops.logreg_block_size(self.observed.size)
            fit = clf.fit_device(self._train, self._labels, out=out[:blk])
            clf.predict_device(self._obs_dev, out=out[blk:])
            host = dev.to_host(out)                      # the one device-to-host read of the round
            fit.set_host(host[:blk])
            fit.check()
            clf._warn_if_not_converged()
            if np.isnan(host[blk]):
                raise ValueError('Input X contains NaN or infinity.')
            return host[blk:]
        X = dev.to_host(self._train)
        return self.predict_log_ratio(X, self._labels_host, self.observed)

    def _process_simulated(self):
        negative_log_ratio_value = -1 * np.asarray(self._log_ratio(), dtype=np.float64)
        self.classifier_attributes += [self.classifier.attributes]
        self.state['n_evidence'] += 1
        parameter_values = self.current_params
        optimize = self._should_optimize()
        self.target_model.update(parameter_values, negative_log_ratio_value, optimize)
        if optimize:
            self.state['last_GP_update'] = self.target_model.n_evidence

    def _should_optimize(self):
        current = self.target_model.n_evidence + 1
        next_update = self.state['last_GP_update'] + self.update_interval
        return current >= self.n_initial_evidence and current >= next_update

    # ---- public -----------------------------------------------------------------------------
    def fit(self, n_evidence, bar=True):
        """Run rounds until the surrogate holds n_evidence points; returns the posterior."""
        logger.info('BOLFIRE: Fitting the surrogate model...')
        if isinstance(n_evidence, int) and n_evidence > 0:
            if n_evidence < self.n_evidence:
                logger.warning('Requesting less evidence than there already exists.')
            return self.infer(n_evidence, bar=bar)
        raise TypeError('n_evidence must be a positive integer.')

    def sample(self, n_samples, warmup=None, n_chains=4, initials=None, algorithm='nuts',
               sigma_proposals=None, n_evidence=None, **kwargs):
        """n_chains NUTS (default) or Metropolis chains of n_samples iterations, warm-up
        included, from the evidence points with the smallest minus log ratio unless `initials`
        (n_chains, n_params) is given; chain i is seeded with get_sub_seed(seed, i).  The chains
        advance in lock-step, one batched GP call per step.  Returns a BOLFIRESample."""
        if self.state['n_batches'] == 0:
            self.fit(n_evidence)
        if algorithm not in ['nuts', 'metropolis']:
            raise ValueError('The given algorithm is not supported.')
        if algorithm == 'metropolis':
            sigma_proposals = resolve_sigmas(self.parameter_names, sigma_proposals,
                                             self.target_model.bounds)
        posterior = self.extract_result()
        warmup = warmup or n_samples // 2
        if initials is not None:
            if np.asarray(initials).shape != (n_chains, self.target_model.input_dim):
                raise ValueError('The shape of initials must be (n_chains, n_params).')
            initials = np.asarray(initials, dtype=float)
        else:
            inds = np.argsort(self.target_model.Y[:, 0])
            initials = np.asarray(self.target_model.X[inds])
        self.target_model.is_sampling = True
        coroutines = []
        start = 0
        for ii in range(n_chains):
            seed = get_sub_seed(self.seed, ii)
            while np.isinf(np.ravel(posterior.logpdf(initials[start]))[0]):
                start += 1
                if start == len(initials):
                    raise ValueError('BOLFIRE.sample: Cannot find enough acceptable '
                                     'initialization points!')
            if algorithm == 'nuts':
                coroutines.append(mcmc.nuts_chain(n_samples, initials[start], n_adapt=warmup,
                                                  seed=seed, **kwargs))
            else:
                coroutines.append(mcmc.metropolis_chain(n_samples, initials[start],
                                                        sigma_proposals, warmup, seed=seed,
                                                        **kwargs))
            start += 1
        chains = np.asarray(mcmc.run_lockstep(coroutines, posterior.logpdf_and_gradient))
        self.target_model.is_sampling = False
        logger.info('{} chains of {} iterations acquired. Effective sample size and Rhat for each '
                    'parameter:'.format(n_chains, n_samples))
        for ii, node in enumerate(self.parameter_names):
            logger.info('{} {} {}'.format(node, mcmc.eff_sample_size(chains[:, :, ii]),
                                          mcmc.gelman_rubin_statistic(chains[:, :, ii])))
        return BOLFIRESample(method_name='BOLFIRE', chains=chains,
                             parameter_names=self.parameter_names, warmup=warmup,
                             n_sim=self.state['n_sim'], seed=self.seed)
