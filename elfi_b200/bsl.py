"""Bayesian synthetic likelihood (Price et al. 2018) with the Gaussian likelihoods on the device.

Host control flow follows the reference (paths relative to elfi-dev/elfi):
  BSL, its Metropolis-Hastings step and logit transform   elfi/methods/inference/bsl.py
  ModelBased (rounds of n_sim_round simulations)          elfi/methods/inference/parameter_inference.py
                                                          (model_based.py, shared with BOLFIRE)
  likelihoods                                             elfi/methods/bsl/pdf_methods.py
  log_SL_stdev, select_penalty, estimate_whitening_matrix elfi/methods/bsl/pre_sample_methods.py
What runs on the device: the simulations of a device model, the (n_sim_round, d) feature matrix
of a round, and the whole likelihood (moments, shrinkage, whitening, Cholesky, log density:
ops.synlik).  The host reads one value per chain and iteration, for the Metropolis-Hastings
step; in throughput mode (device_proposal) the step runs on the device too (ops.bsl_mh_step) and
hands the simulator device columns.  The pre-sample tools evaluate all M simulation sets, and all
penalties, in one call.

The standard (Warton-shrunk, whitened) and unbiased Gaussian likelihoods are provided.
semiBSL, the R-BSL adjustments and graphical-lasso shrinkage raise NotImplementedError.  Any other
callable likelihood is called on the host with NumPy (ssx, ssy).
"""
import logging

import numpy as np
import scipy.linalg
import torch

from . import device as dev
from . import mcmc
from . import model as em
from . import ops
from .results import BslSample
from .model_based import ModelBased, feature_columns, feature_list, observed_row
from .samplers import ModelPrior

logger = logging.getLogger(__name__)

__all__ = ['BSL', 'standard_likelihood', 'unbiased_likelihood', 'semiparametric_likelihood',
           'robust_likelihood', 'gaussian_syn_likelihood', 'gaussian_syn_likelihood_ghurye_olkin',
           'log_SL_stdev', 'select_penalty', 'estimate_whitening_matrix']


# ------------------------------------------------------------------------------- likelihoods
class SyntheticLikelihood:
    """A Gaussian synthetic likelihood evaluated by ops.synlik: estimator 'standard' (optional
    Warton penalty and whitening matrix) or 'unbiased'.  Called with (ssx, ssy) it returns
    np.array([ll]) like the reference's likelihoods; ``device`` keeps the result on the device."""

    def __init__(self, estimator='standard', penalty=None, whitening=None):
        if penalty is not None and not 0 <= penalty <= 1:
            raise ValueError('The Warton penalty must lie in [0, 1], got {}'.format(penalty))
        self.estimator = estimator
        self.penalty = penalty
        self.whitening = whitening
        self._w_dev = None

    def device(self, ssx, ssy, penalties=None):
        """ll of each group of ssx ((n, d) or (G, n, d)) as a device tensor (G,), or (G, K) for
        the K `penalties` given here in place of this likelihood's own."""
        if self.whitening is not None and self._w_dev is None:
            self._w_dev = dev.to_device(np.asarray(self.whitening, dtype=np.float64))
        pen = penalties if penalties is not None else \
            (None if self.penalty is None else [self.penalty])
        ll = ops.synlik(ssx, ssy, estimator=self.estimator, penalties=pen, whitening=self._w_dev)
        return ll if penalties is not None else ll.reshape(-1)

    def __call__(self, ssx, ssy):
        return np.array([float(self.device(ssx, ssy)[0].item())])

    def __repr__(self):
        return 'SyntheticLikelihood({!r}, penalty={}, whitening={})'.format(
            self.estimator, self.penalty, None if self.whitening is None else 'W')


def standard_likelihood(shrinkage=None, penalty=None, whitening=None, standardise=False):
    """The standard Gaussian synthetic likelihood, with Warton shrinkage (shrinkage='warton' and a
    penalty in [0, 1]) and whitening by a (d, d) matrix, both optional.  `standardise` belongs to
    graphical-lasso shrinkage, which is not provided."""
    if shrinkage == 'glasso':
        raise NotImplementedError("shrinkage='glasso' (graphical lasso) is not provided; use "
                                  "shrinkage='warton' or none")
    if shrinkage not in (None, 'warton'):
        raise ValueError("shrinkage must be None or 'warton', got {!r}".format(shrinkage))
    if shrinkage == 'warton':
        if penalty is None:
            raise ValueError("shrinkage='warton' needs a penalty in [0, 1]")
        return SyntheticLikelihood('standard', float(np.reshape(penalty, -1)[0]), whitening)
    return SyntheticLikelihood('standard', None, whitening)


def unbiased_likelihood():
    """The unbiased Gaussian synthetic likelihood of Ghurye and Olkin (1969)."""
    return SyntheticLikelihood('unbiased')


def semiparametric_likelihood(shrinkage=None, penalty=None, whitening=None):
    raise NotImplementedError('semiBSL (semiparametric_likelihood: the KDE marginals and the '
                              'Gaussian copula) is not provided')


def robust_likelihood(adjustment):
    raise NotImplementedError('R-BSL (robust_likelihood, the {!r} adjustment and its slice '
                              'sampler) is not provided'.format(adjustment))


def semi_param_kernel_estimate(ssx, ssy, shrinkage=None, penalty=None, whitening=None):
    semiparametric_likelihood()


def syn_likelihood_misspec(ssx, ssy, gamma, adjustment):
    robust_likelihood(adjustment)


def gaussian_syn_likelihood(ssx, ssy, shrinkage=None, penalty=None, whitening=None,
                            standardise=False):
    """np.array([ll]): the standard synthetic log-likelihood of ssy under the simulated summaries
    ssx (n, d), computed on the device (see standard_likelihood)."""
    return standard_likelihood(shrinkage, penalty, whitening, standardise)(ssx, ssy)


def gaussian_syn_likelihood_ghurye_olkin(ssx, ssy):
    """np.array([ll]): the unbiased synthetic log-likelihood, computed on the device."""
    return unbiased_likelihood()(ssx, ssy)


def _device_likelihood(likelihood):
    """The SyntheticLikelihood a likelihood argument stands for, or None for a host callable."""
    if likelihood is None or likelihood is gaussian_syn_likelihood:
        return SyntheticLikelihood('standard')
    if likelihood is gaussian_syn_likelihood_ghurye_olkin:
        return SyntheticLikelihood('unbiased')
    if isinstance(likelihood, SyntheticLikelihood):
        return likelihood
    return None


# ------------------------------------------------------------------------------- features
def _simulate_features(model, n_sim, feature_names, params, seed):
    """(n_sim, d) device matrix of the features simulated at params (model.generate)."""
    out = model.generate(n_sim, outputs=list(feature_names), with_values=params, seed=seed)
    blocks = feature_columns(out, feature_names, n_sim)
    return blocks[0] if len(blocks) == 1 else torch.cat(blocks, dim=1)


def _param_values(model, theta):
    return theta if isinstance(theta, dict) else dict(zip(model.parameter_names, theta))


# ------------------------------------------------------------------------------- sampler
class BSL(ModelBased):
    """Bayesian synthetic likelihood with a random-walk Metropolis-Hastings sampler (Price et al.
    2018).  Each round simulates n_sim_round times at one parameter; the round's features stay on
    the device and go to one likelihood call.  Runs on this rank only.

    Several chains (``sample(..., n_chains=C)``) run in lock-step: each batch holds batch_size rows
    of every chain, and one likelihood call evaluates the C rounds of an iteration.
    ``device_proposal`` (throughput mode, e.g. ``DeviceModelPrior(m)``: an object with the (p, 5)
    prior table ``specs``, its ``sources`` and ``logpdf``) moves the proposals, the prior
    densities, the Metropolis-Hastings decisions and the chains to the device
    (ops.bsl_mh_step), so that the host only launches work; its chains follow the same sampler
    from a Philox stream rather than the host RandomState."""

    D_MAX = ops.SYNLIK_D_MAX

    def __init__(self, model, n_sim_round, feature_names=None, likelihood=None, batch_size=None,
                 seed=None, pool=None, device_proposal=None):
        super().__init__(model, n_sim_round, feature_names=feature_names, batch_size=batch_size,
                         seed=seed, pool=pool)
        self.random_state = np.random.RandomState(self.seed)
        self.likelihood = likelihood
        self._device_lik = _device_likelihood(likelihood)
        if device_proposal is not None and self._device_lik is None:
            raise ValueError('device_proposal keeps the chains on the device and needs a device '
                             'likelihood (standard or unbiased), not a host callable')
        self.device_proposal = device_proposal
        self._obs_dev = None
        self.param_names = None
        self.prior = None
        self.sigma_proposals = None
        self.burn_in = 0
        self.logit_transform_bound = None

    @property
    def parameter_names(self):
        return self.param_names or self.model.parameter_names

    def sample(self, n_samples, sigma_proposals, params0=None, param_names=None, burn_in=0,
               logit_transform_bound=None, n_chains=1):
        """Run n_chains chains of n_samples iterations (burn-in included) from params0 ((p,) for
        every chain, or (n_chains, p); a prior draw per chain by default) with Gaussian random-walk
        proposals of covariance sigma_proposals, in the logit-transformed space when
        logit_transform_bound ((p, 2) lower and upper bounds) is given.  Chain 0 draws its
        proposals and uniforms from RandomState(seed), chain c >= 1 from
        RandomState(get_sub_seed(seed, c)).  Returns a BslSample; with n_chains > 1 it also holds
        `chains` (n_chains, n_samples, p) and the per-chain `acc_rates`."""
        self._set_up(n_samples, sigma_proposals, params0, param_names, burn_in,
                     logit_transform_bound, n_chains)
        return self.infer(n_samples)

    def _set_up(self, n_samples, sigma_proposals, params0=None, param_names=None, burn_in=0,
                logit_transform_bound=None, n_chains=1, device_state=None):
        """Everything `sample` does before its rounds: the prior, the chains, the initial state and,
        in throughput mode, the device chains (in `device_state` when given, see
        _init_device_chains).  A Testbench sets up several samplers this way and runs their rounds
        together."""
        n_chains = int(n_chains)
        if n_chains < 1:
            raise ValueError('n_chains must be at least 1, got {}'.format(n_chains))
        if n_chains > 1 and self.pool is not None:
            raise ValueError('BSL with n_chains > 1 does not store its batches in a pool')
        self.sigma_proposals = sigma_proposals
        self.param_names = param_names
        self.prior = ModelPrior(self.model, parameter_names=self.parameter_names)
        self.burn_in = burn_in
        self.logit_transform_bound = None if logit_transform_bound is None else \
            np.array(logit_transform_bound)
        self._set_chains(n_chains)
        self._init_state(n_samples, params0, device_state)

    def _set_chains(self, C):
        if C != self.n_chains:
            self._sim = None
        self.n_chains = C
        self.computation_context.batch_size = C * self._rows_per_chain
        self._random_states = [self.random_state] + [
            np.random.RandomState(em.get_sub_seed(self.seed, c)) for c in range(1, C)]

    def _initial_points(self, params0):
        """(C, p) host starting points, each inside the prior support."""
        C, p = self.n_chains, len(self.parameter_names)
        if params0 is None:
            drawn = self.model.generate(C, self.parameter_names, seed=self.seed)
            return np.column_stack([dev.to_host(drawn[q]) for q in self.parameter_names])
        params0 = np.array(params0, dtype=float)
        if params0.size == p:
            params0 = np.broadcast_to(params0.reshape(1, p), (C, p)).copy()
        if params0.shape != (C, p):
            raise ValueError('params0 must be ({0},) or ({1}, {0}), got shape {2}'.format(
                p, C, params0.shape))
        outside = ~np.isfinite(np.reshape(self.prior.logpdf(params0), -1))
        if outside.any():
            where = '' if C == 1 else ' (chain {})'.format(
                ', '.join(str(c) for c in np.flatnonzero(outside)))
            raise ValueError('Initial point {} is outside prior support{}.'.format(
                params0[outside][0] if C > 1 else params0[0], where))
        return params0

    def _init_state(self, n_samples, params0=None, device_state=None):
        self.state['n_batches'] = 0
        self.state['n_sim'] = 0
        self.state['round'] = 0
        self.state['n_sim_round'] = 0
        self.state['n_samples'] = 0
        C, p = self.n_chains, len(self.parameter_names)
        params0 = self._initial_points(params0)
        # (C, n_samples, ...) host state; state[...] shows chain 0 alone when C = 1
        self._params = np.zeros((C, n_samples, p))
        self._logprior = np.zeros((C, n_samples))
        self._logpost = np.zeros((C, n_samples))
        self._n_acc = np.zeros(C, dtype=np.int64)
        self._live = np.ones(C, dtype=bool)
        self._params[:, 0] = params0
        self._logprior[:, 0] = np.reshape(self.prior.logpdf(params0), -1)
        self._share_state()
        if self.device_proposal is not None:
            self._init_device_chains(n_samples, params0, device_state)

    def _share_state(self):
        one = (lambda a: a[0]) if self.n_chains == 1 else (lambda a: a)
        self.state['params'] = one(self._params)
        self.state['logprior'] = one(self._logprior)
        self.state['logposterior'] = one(self._logpost)

    def _init_device_chains(self, n_samples, params0, device_state=None):
        """Device state of throughput mode: the chains, their log posteriors and acceptance
        counters, the pending proposals (params0 at iteration 0) and the (p, C b) parameters of
        the next batch.  `device_state` may hold zero-filled views of caller-owned buffers of
        these shapes under the keys 'chains', 'logpost', 'n_acc', 'prop', 'prop_lp' and 'rows'
        (a column block of a wider (p, .) matrix); otherwise this sampler allocates its own."""
        dp = self.device_proposal
        names = list(self.parameter_names)
        if list(dp.parameter_names) != names:
            raise ValueError('device_proposal has the parameters {}, the sampler {}'.format(
                list(dp.parameter_names), names))
        C, p, b = self.n_chains, len(names), self._rows_per_chain
        sources = dp.sources if getattr(dp, '_cond', False) else None
        self._tables = ops.bsl_mh_tables(dp.specs, self.sigma_proposals, sources,
                                         self.logit_transform_bound)
        if device_state is None:
            self._prop = dev.to_device(params0).contiguous()
            self._prop_lp = dp.logpdf(self._prop)
            self._chains_dev = dev.zeros((C, n_samples, p))
            self._logpost_dev = dev.zeros((C, n_samples))
            self._n_acc_dev = dev.zeros((C,), dtype=torch.int64)
            self._rows = dev.empty((p, C * b))
        else:
            self._prop = device_state['prop']
            self._prop.copy_(dev.to_device(params0))
            self._prop_lp = device_state['prop_lp']
            self._prop_lp.copy_(dp.logpdf(self._prop))
            self._chains_dev = device_state['chains']
            self._logpost_dev = device_state['logpost']
            self._n_acc_dev = device_state['n_acc']
            self._rows = device_state['rows']
        self._rows.view(p, C, b).copy_(self._prop.t()[:, :, None].expand(p, C, b))

    def prepare_new_batch(self, batch_index):
        if self.device_proposal is None:
            return super().prepare_new_batch(batch_index)
        return {q: self._rows[i] for i, q in enumerate(self.parameter_names)}

    @property
    def current_params(self):
        return self._params[:, self.state['n_samples']]

    def _rounds(self):
        return self._sim if self._sim.dim() == 3 else self._sim[None]

    def _loglikelihoods(self):
        """(C,) log-likelihoods of the rounds of the chains that simulated their proposal: a device
        tensor for a device likelihood (one call with G = C), else a host array (NaN for the
        other chains)."""
        if self._device_lik is not None:
            if self._obs_dev is None:
                self._obs_dev = dev.to_device(self.observed.reshape(-1))
            return self._device_lik.device(self._rounds(), self._obs_dev)
        sims = dev.to_host(self._rounds())
        ll = np.full(self.n_chains, np.nan)
        for c in np.flatnonzero(self._live):
            sim = sims[c]
            ll[c] = -np.inf if not np.all(np.isfinite(sim)) else \
                float(np.reshape(self.likelihood(sim, self.observed), -1)[0])
        return ll

    def _check_first_round(self, ll):
        bad = np.flatnonzero(~np.isfinite(ll))
        if len(bad):
            where = '' if self.n_chains == 1 else ' (chain {})'.format(
                ', '.join(str(c) for c in bad))
            raise RuntimeError('Estimated likelihood not finite on initialisation round{}.'.format(
                where))

    def _process_simulated(self):
        self._step(self._loglikelihoods())

    def _step(self, ll):
        """The Metropolis-Hastings step of the round, from the (C,) log-likelihoods of
        `_loglikelihoods` (or the same values computed by a caller)."""
        n = self.state['n_samples']
        if self.device_proposal is not None:
            if n == 0:
                self._check_first_round(dev.to_host(ll))   # the one read of throughput mode
            ops.bsl_mh_step(self._tables, n, ll, self._prop, self._prop_lp, self._chains_dev,
                            self._logpost_dev, self._n_acc_dev, self._rows, int(self.seed),
                            self.burn_in)
            self.state['n_samples'] += 1
            return
        if dev.is_device_array(ll):
            ll = dev.to_host(ll)          # the one device-to-host read of the iteration
        if n == 0:
            self._check_first_round(ll)
        if not np.all(np.isfinite(ll[self._live])):
            logger.warning('Estimated likelihood not finite.')
        for c in np.flatnonzero(self._live):
            self._logpost[c, n] = ll[c] + self._logprior[c, n]
            if n == 0:
                accept = True
            else:
                prob = np.minimum(1.0, self._get_mh_ratio(c))
                accept = self._random_states[c].uniform() < prob
            if accept:
                if n >= self.burn_in:
                    self._n_acc[c] += 1
            else:
                self._copy_previous(n, c)
        self.state['n_samples'] += 1

    def _copy_previous(self, n, chains):
        for arr in (self._logprior, self._params, self._logpost):
            arr[chains, n] = arr[chains, n - 1]

    def _init_round(self):
        """Propose the next parameter of every chain.  A chain whose proposal is outside the prior
        support keeps its state for this iteration and simulates its rows at it; when every
        chain's proposal is outside, nothing is simulated and the remaining objective shortens by
        one round."""
        if self.device_proposal is not None:
            self.state['n_sim_round'] = 0          # ops.bsl_mh_step wrote the next parameters
            return
        while self.state['n_samples'] < self._params.shape[1]:
            n = self.state['n_samples']
            props = np.vstack([self._propagate_state(c) for c in range(self.n_chains)])
            logprior = np.reshape(self.prior.logpdf(props), -1)
            live = np.isfinite(logprior)
            self._live = live
            self._copy_previous(n, ~live)
            self._params[live, n] = props[live]
            self._logprior[live, n] = logprior[live]
            if live.any():
                self.state['n_sim_round'] = 0
                break
            self.state['n_samples'] += 1
            self.set_objective(self.objective['round'] - 1)

    def _propagate_state(self, c):
        mean = self._params[c, self.state['n_samples'] - 1]
        random_state = self._random_states[c]
        bound = self.logit_transform_bound
        if bound is None:
            return random_state.multivariate_normal(mean, self.sigma_proposals)
        return self._para_logit_back_transform(random_state.multivariate_normal(
            self._para_logit_transform(mean, bound), self.sigma_proposals), bound)

    def _get_mh_ratio(self, c):
        n = self.state['n_samples']
        params, logpost = self._params[c], self._logpost[c]
        log_ratio = logpost[n] - logpost[n - 1]
        jac = 0
        if self.logit_transform_bound is not None:
            # the Jacobian terms are evaluated at the parameters themselves, as in the reference
            jac = self._jacobian_logit_transform(params[n], self.logit_transform_bound) \
                - self._jacobian_logit_transform(params[n - 1], self.logit_transform_bound)
        res = jac + log_ratio
        return np.exp(min(700, max(-700, res)))

    # bound kinds: 0 both bounds finite, 1 lower infinite, 2 upper infinite, 3 both infinite
    @staticmethod
    def _bound_kinds(bound):
        inf = np.isinf(np.asarray(bound, dtype=float))
        return inf[:, 0] * 1 + inf[:, 1] * 2

    @staticmethod
    def _para_logit_transform(theta, bound):
        """theta -> the unbounded proposal space: log((x - a) / (b - x)), log(1 / (b - x)),
        log(x - a) or x, by which of the bounds (a, b) are finite."""
        theta = np.asarray(theta, dtype=float).flatten()
        kinds = BSL._bound_kinds(bound)
        out = np.zeros(len(theta))
        for i, (x, kind) in enumerate(zip(theta, kinds)):
            a, b = bound[i, 0], bound[i, 1]
            if kind == 0:
                out[i] = np.log((x - a) / (b - x))
            elif kind == 1:
                out[i] = np.log(1 / (b - x))
            elif kind == 2:
                out[i] = np.log(x - a)
            else:
                out[i] = x
        return out

    @staticmethod
    def _para_logit_back_transform(theta_tilde, bound):
        """The inverse of _para_logit_transform."""
        theta_tilde = np.asarray(theta_tilde, dtype=float).flatten()
        kinds = BSL._bound_kinds(bound)
        out = np.zeros(len(theta_tilde))
        for i, (y, kind) in enumerate(zip(theta_tilde, kinds)):
            a, b = bound[i, 0], bound[i, 1]
            ey = np.exp(y)
            if kind == 0:
                out[i] = a / (1 + ey) + b / (1 + (1 / ey))
            elif kind == 1:
                out[i] = b - (1 / ey)
            elif kind == 2:
                out[i] = a + ey
            else:
                out[i] = y
        return out

    @staticmethod
    def _jacobian_logit_transform(theta_tilde, bound):
        """log |d theta / d theta_tilde| of the back transform, summed over the parameters."""
        theta_tilde = np.asarray(theta_tilde, dtype=float).flatten()
        kinds = BSL._bound_kinds(bound)
        logj = np.zeros(len(theta_tilde))
        for i, (y, kind) in enumerate(zip(theta_tilde, kinds)):
            if kind == 0:
                a, b = bound[i, 0], bound[i, 1]
                ey = np.exp(y)
                logj[i] = np.log(b - a) - np.log((1 / ey) + 2 + ey)
            elif kind in (1, 2):
                logj[i] = y
        return np.sum(logj)

    def extract_result(self):
        if self.device_proposal is not None:
            # the one read of the device chains, at the end of the run
            self._params[:] = dev.to_host(self._chains_dev)
            self._logpost[:] = dev.to_host(self._logpost_dev)
            self._n_acc[:] = dev.to_host(self._n_acc_dev)
            self.state.pop('logprior', None)
        n_kept = self.state['n_samples'] - self.burn_in
        if self.n_chains == 1:
            self.num_accepted = int(self._n_acc[0])
            samples_all = {p: np.array(self._params[0, :, i])
                           for i, p in enumerate(self.parameter_names)}
            acc_rate = self.num_accepted / n_kept
            logger.info('MCMC acceptance rate: {}'.format(acc_rate))
            return BslSample(method_name='BSL', samples_all=samples_all, acc_rate=acc_rate,
                             burn_in=self.burn_in, n_sim=self.state['n_sim'],
                             parameter_names=self.parameter_names)
        chains = np.array(self._params)
        self.num_accepted = int(self._n_acc.sum())
        acc_rate = self.num_accepted / (self.n_chains * n_kept)
        logger.info('MCMC acceptance rate: {} ({} chains)'.format(acc_rate, self.n_chains))
        logger.info('{} chains of {} iterations acquired. Effective sample size and Rhat for each '
                    'parameter:'.format(self.n_chains, chains.shape[1]))
        for i, name in enumerate(self.parameter_names):
            kept = chains[:, self.burn_in:, i]
            logger.info('{} {} {}'.format(name, mcmc.eff_sample_size(kept),
                                          mcmc.gelman_rubin_statistic(kept)))
        return BslSample(method_name='BSL',
                         samples_all={p: chains[:, :, i] for i, p in enumerate(self.parameter_names)},
                         acc_rate=acc_rate, burn_in=self.burn_in, n_sim=self.state['n_sim'],
                         parameter_names=self.parameter_names, chains=chains,
                         acc_rates=self._n_acc / n_kept, n_chains=self.n_chains)


# ------------------------------------------------------------------------------- pre-sample tools
def _simulation_sets(model, n_sim, feature_names, params, seed, M):
    """(M, n_sim, d) device features of M simulation sets, set i from the i-th child seed of
    SeedSequence(seed)."""
    child_seeds = np.random.SeedSequence(seed).generate_state(M)
    return torch.stack([_simulate_features(model, n_sim, feature_names, params, s)
                        for s in child_seeds])


def log_SL_stdev(model, theta, n_sim, feature_names, likelihood=None, M=20, seed=None):
    """Standard deviation of the log synthetic likelihood at theta over M simulation sets, for
    each simulation count in n_sim.  A device likelihood evaluates the M sets in one call per
    count."""
    params = _param_values(model, theta)
    feature_names = feature_list(feature_names)
    observed = observed_row(model, feature_names)
    n_sim = np.atleast_1d(n_sim)
    sets = _simulation_sets(model, int(max(n_sim)), feature_names, params, seed, M)
    lik = _device_likelihood(likelihood)
    ll = np.zeros((len(n_sim), M))
    for n_i, n in enumerate(n_sim):
        if lik is not None:
            ll[n_i] = dev.to_host(lik.device(sets[:, :int(n)], observed.reshape(-1)))
        else:
            host = dev.to_host(sets)
            for i in range(M):
                ll[n_i, i] = np.reshape(likelihood(host[i, :int(n)], observed), -1)[0]
    return np.std(ll, axis=1)


def select_penalty(model, n_sim, theta, feature_names, likelihood=None, lmdas=None, M=20,
                   sigma=1.5, shrinkage='glasso', whitening=None, seed=None, verbose=False):
    """The Warton penalty, per simulation count in n_sim, whose log synthetic likelihood standard
    deviation over M simulation sets is closest to sigma.  Returns (penalties, standard
    deviations).  With the default likelihood all M sets and all penalties of one simulation
    count are one device call.  shrinkage='glasso' (the reference's default) is not provided."""
    if shrinkage == 'glasso':
        raise NotImplementedError("select_penalty: shrinkage='glasso' (graphical lasso) is not "
                                  "provided; pass shrinkage='warton'")
    if shrinkage != 'warton':
        raise ValueError("shrinkage must be 'warton', got {!r}".format(shrinkage))
    params = _param_values(model, theta)
    feature_names = feature_list(feature_names)
    ssy = observed_row(model, feature_names)
    if lmdas is None:
        lmdas = list(np.arange(0.2, 0.8, 0.02))
    lmdas = list(lmdas)
    batch_size = np.array([n_sim]).flatten()
    ns, n_lambda = len(batch_size), len(lmdas)
    sets = _simulation_sets(model, int(max(batch_size)), feature_names, params, seed, M)
    logliks = np.zeros((M, ns, n_lambda))
    on_device = likelihood is None or likelihood is gaussian_syn_likelihood
    if on_device:
        lik = SyntheticLikelihood('standard', None, whitening)
    for n_i, n in enumerate(batch_size):
        if on_device:
            logliks[:, n_i, :] = dev.to_host(lik.device(sets[:, :int(n)], ssy.reshape(-1),
                                                        penalties=lmdas))
        else:
            host = dev.to_host(sets)
            for m in range(M):
                for k, lmda in enumerate(lmdas):
                    logliks[m, n_i, k] = np.reshape(likelihood(
                        host[m, :int(n)], ssy, shrinkage=shrinkage, penalty=lmda,
                        whitening=whitening), -1)[0]
    closest_lmdas = np.zeros(ns)
    closest_std_devs = np.zeros(ns)
    for i in range(ns):
        std_devs = np.array([np.std(logliks[:, i, j]) for j in range(n_lambda)])
        best = np.argmin(np.abs(std_devs - sigma))
        closest_lmdas[i] = lmdas[best]
        closest_std_devs[i] = std_devs[best]
        if verbose:
            print('n_sim {}: logliks {}, std_devs {}'.format(batch_size[i], logliks[:, i],
                                                            std_devs))
    return closest_lmdas, closest_std_devs


def estimate_whitening_matrix(model, n_sim, theta, feature_names, likelihood_type='standard',
                              seed=None):
    """Whitening matrix W (d, d) of Priddle et al. (2021) from n_sim simulations at theta: the
    eigen-decomposition of the correlation of the standardised features, W = diag(w^-1/2) V^T,
    both factors rounded to 8 decimals.  Host arithmetic (one d x d set-up), so W is the same
    bits for the same simulations."""
    if likelihood_type not in ('standard', 'semiparametric'):
        raise ValueError("Unsupported likelihood type '{}'.".format(likelihood_type))
    if likelihood_type == 'semiparametric':
        raise NotImplementedError("estimate_whitening_matrix: likelihood_type='semiparametric' "
                                  "(semiBSL) is not provided")
    params = _param_values(model, theta)
    feature_names = feature_list(feature_names)
    ssx = dev.to_host(_simulate_features(model, n_sim, feature_names, params, seed))
    centred = ssx - np.mean(ssx, axis=0)
    standardised = centred / np.std(ssx, axis=0)
    eigval, eigvec = scipy.linalg.eig(np.cov(np.transpose(standardised)))
    scale = np.diag(np.power(eigval, -0.5)).real.round(8)
    return np.dot(scale, eigvec.T).real.round(8)
