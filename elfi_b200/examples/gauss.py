"""Gaussian noise model (mirror of elfi/examples/gauss.py, 1-d case) with device summaries."""
from functools import partial

import numpy as np
import scipy.stats as ss

from .. import model as em
from .. import ops
from ..throughput import LazySimulation, batch_columns, batch_key

# the key draw under its earlier name, which tests/device_prior_cases.py seeds its simulator with
_key = batch_key


def gauss(mu, sigma, n_obs=50, batch_size=1, random_state=None):
    """elfi/examples/gauss.py:11-35."""
    batches_mu = np.asanyarray(mu).reshape((-1, 1))
    batches_sigma = np.asanyarray(sigma).reshape((-1, 1))
    return ss.norm.rvs(loc=batches_mu, scale=batches_sigma, size=(batch_size, n_obs),
                       random_state=random_state)


def ss_mean(y):
    """np.mean(y, axis=1) on the device (elfi/examples/gauss.py:142-156)."""
    return y.summaries()[:, 0] if isinstance(y, LazySimulation) else ops.meanvar(y)[:, 0]


def ss_var(y):
    """np.var(y, axis=1) on the device (elfi/examples/gauss.py:159-173)."""
    return y.summaries()[:, 1] if isinstance(y, LazySimulation) else ops.meanvar(y)[:, 1]


def _prior_params(true_params):
    """[mu_lo, mu_width, a, b] of the priors uniform(mu_lo, mu_width) of mu and truncnorm(a, b) of
    sigma."""
    eps_prior = 5
    return [true_params[0] - eps_prior, 2 * eps_prior,
            np.amax([.01, true_params[1] - eps_prior]), 2 * eps_prior]


def _graph(m, uniform, truncnorm, prm, simulator, y_obs):
    """Priors, simulator, summaries and distance of elfi/examples/gauss.py:75-139."""
    priors = [em.Prior(uniform, prm[0], prm[1], model=m, name='mu'),
              em.Prior(truncnorm, prm[2], prm[3], model=m, name='sigma')]
    em.Simulator(simulator, *priors, observed=y_obs, name='gauss')
    sumstats = [em.Summary(ss_mean, m['gauss'], name='ss_mean'),
                em.Summary(ss_var, m['gauss'], name='ss_var')]
    em.Distance('euclidean', *sumstats, name='d')
    return m


def get_model(n_obs=50, true_params=None, seed_obs=None):
    """elfi/examples/gauss.py:75-139 (nd_mean=False)."""
    if true_params is None:
        true_params = [4, .4]
    y_obs = gauss(*true_params, n_obs=n_obs, random_state=np.random.RandomState(seed_obs))
    return _graph(em.new_model(), 'uniform', 'truncnorm', _prior_params(true_params),
                  partial(gauss, n_obs=n_obs), y_obs)


# ---------------------------------------------------------------------------- throughput mode
# Device-side priors, simulator fused with its mean / variance summaries, and proposals
# (Philox streams; statistical parity with the host path).  See examples/ma2.py for the design.
def gauss_device(mu, sigma, n_obs=50, batch_size=1, random_state=None):
    """Device twin of gauss with the mean and variance fused into the simulator; returns a
    LazySimulation."""
    mu, sigma = batch_columns((mu, sigma), batch_size)
    key = batch_key(random_state)
    return LazySimulation(
        (int(mu.numel()), n_obs),
        lambda kind: ops.sim_gauss(mu, sigma, n_obs, seed=key)[1],
        lambda: ops.sim_gauss(mu, sigma, n_obs, seed=key, want_data=True, want_summaries=False)[0])


class DeviceProposal:
    """SMC proposals / prior density on the device for the Gaussian model
    (pass an instance as ``device_proposal=`` to SMC)."""
    parameter_names = ['mu', 'sigma']

    def __init__(self, prm):
        self.prm = list(prm)                      # [mu_lo, mu_width, a, b]
        self.box = ([prm[0], prm[2]], [prm[0] + prm[1], prm[3]])

    def rvs(self, means, cov, weights, size, key, cdf=None):
        return ops.gm_rvs(means, cov, weights, size, seed=key, support=2, box=self.box, cdf=cdf)

    def logpdf(self, params):
        return ops.logprior_gauss(params, self.prm)


class _DeviceUniform:
    """uniform(loc, scale) prior of mu with device draws (pdf/logpdf as scipy's)."""

    @staticmethod
    def rvs(loc, scale, size=1, random_state=None):
        n = int(np.prod(size))
        u = ops.prior_gauss(n, batch_key(random_state), [0.0, 1.0, 0.0, 1.0])[0]
        return loc + scale * u

    pdf = staticmethod(lambda x, loc, scale: ss.uniform.pdf(x, loc, scale))
    logpdf = staticmethod(lambda x, loc, scale: ss.uniform.logpdf(x, loc, scale))


class _DeviceTruncnorm:
    """truncnorm(a, b) prior of sigma with device draws."""

    @staticmethod
    def rvs(a, b, size=1, random_state=None):
        n = int(np.prod(size))
        return ops.prior_gauss(n, batch_key(random_state), [0.0, 1.0, a, b])[1]

    pdf = staticmethod(lambda x, a, b: ss.truncnorm.pdf(x, a, b))
    logpdf = staticmethod(lambda x, a, b: ss.truncnorm.logpdf(x, a, b))


def get_device_model(n_obs=50, true_params=None, seed_obs=None):
    """Gaussian noise inference task with priors, simulator and summaries on the device.
    Returns (model, DeviceProposal instance)."""
    if true_params is None:
        true_params = [4, .4]
    y_obs = gauss(*true_params, n_obs=n_obs, random_state=np.random.RandomState(seed_obs))
    prm = _prior_params(true_params)
    m = _graph(em.new_model(), _DeviceUniform, _DeviceTruncnorm, prm,
               partial(gauss_device, n_obs=n_obs), y_obs)
    return m, DeviceProposal(prm)
