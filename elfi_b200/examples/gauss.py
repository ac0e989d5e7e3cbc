"""Gaussian noise models (mirror of elfi/examples/gauss.py) with device summaries: the 1-D model of
mu and sigma, and the n-D mean model (nd_mean=True) of D means mu_0 .. mu_{D-1} under a fixed
covariance, whose summaries are the per-coordinate means and variances and whose distance is
euclidean_multidim of the means.

The host paths (gauss, gauss_nd_mean, get_model) consume the batch's RandomState exactly as the
reference does, so they reproduce the reference's draws; get_device_model is the same task in
throughput mode (Philox streams; statistical parity with the host path).
"""
from functools import partial

import numpy as np
import scipy.stats as ss

from .. import device as dev
from .. import model as em
from .. import ops
from ..priors import DeviceModelPrior
from ..throughput import LazySimulation, batch_columns, batch_key

# the key draw under its earlier name, which tests/device_prior_cases.py seeds its simulator with
_key = batch_key


def gauss(mu, sigma, n_obs=50, batch_size=1, random_state=None):
    """elfi/examples/gauss.py:11-35."""
    batches_mu = np.asanyarray(mu).reshape((-1, 1))
    batches_sigma = np.asanyarray(sigma).reshape((-1, 1))
    return ss.norm.rvs(loc=batches_mu, scale=batches_sigma, size=(batch_size, n_obs),
                       random_state=random_state)


def gauss_nd_mean(*mu, cov_matrix, n_obs=15, batch_size=1, random_state=None):
    """elfi/examples/gauss.py:38-72: (batch_size, n_obs, D) draws of the D-dimensional normal with
    means mu and covariance cov_matrix, one SciPy multivariate_normal call per row."""
    n_dim = len(mu)
    batches_mu = np.zeros(shape=(batch_size, n_dim))
    for idx_dim, param_mu in enumerate(mu):
        batches_mu[:, idx_dim] = param_mu
    y_obs = np.zeros(shape=(batch_size, n_obs, n_dim))
    for idx_batch in range(batch_size):
        y_batch = ss.multivariate_normal.rvs(mean=batches_mu[idx_batch], cov=cov_matrix,
                                             size=n_obs, random_state=random_state)
        if n_dim == 1:
            y_batch = y_batch[:, np.newaxis]
        y_obs[idx_batch, :, :] = y_batch
    return y_obs


def _nd_summaries(y):
    """[means | variances] (B, 2 D) of rank-3 data: the fused columns of a lazy output, else the
    device summary kernel; None for rank-2 data."""
    if isinstance(y, LazySimulation):
        return y.summaries() if y.ndim == 3 else None
    if (y.dim() if dev.is_device_array(y) else np.ndim(y)) == 3:
        return ops.gauss_nd_summaries(y)
    return None


def ss_mean(y):
    """np.mean(y, axis=1) on the device (elfi/examples/gauss.py:142-156): (B,) for (B, n) data,
    (B, D) for (B, n, D) data."""
    S = _nd_summaries(y)
    if S is not None:
        return S[:, :S.shape[1] // 2]
    return y.summaries()[:, 0] if isinstance(y, LazySimulation) else ops.meanvar(y)[:, 0]


def ss_var(y):
    """np.var(y, axis=1) on the device (elfi/examples/gauss.py:159-173): (B,) for (B, n) data,
    (B, D) for (B, n, D) data."""
    S = _nd_summaries(y)
    if S is not None:
        return S[:, S.shape[1] // 2:]
    return y.summaries()[:, 1] if isinstance(y, LazySimulation) else ops.meanvar(y)[:, 1]


def euclidean_multidim(*simulated, observed):
    """elfi/examples/gauss.py:176-198: the Euclidean distance of the first summary to its observed
    value (the other summaries are not used, as in the reference).  Device summaries give a device
    (B,) result (ops.gauss_nd_distance, NumPy's order); host arrays run the reference's NumPy."""
    pts_sim = simulated[0]
    pts_obs = observed[0]
    if dev.is_device_array(pts_sim):
        return ops.gauss_nd_distance(pts_sim, pts_obs)
    d_dim_merged = np.sum((pts_sim - pts_obs)**2., axis=1)
    return np.sqrt(d_dim_merged)


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


def _graph_nd(m, priors, simulator, y_obs):
    """Priors mu_0 .. mu_{D-1}, simulator, summaries and distance of gauss.py:96-139 (nd_mean)."""
    eps_prior = 5
    pr = [em.Prior(prior, loc - eps_prior, 2 * eps_prior, model=m, name='mu_{}'.format(i))
          for i, (prior, loc) in enumerate(priors)]
    em.Simulator(simulator, *pr, observed=y_obs, name='gauss')
    sumstats = [em.Summary(ss_mean, m['gauss'], name='ss_mean'),
                em.Summary(ss_var, m['gauss'], name='ss_var')]
    em.Discrepancy(euclidean_multidim, *sumstats, name='d')
    return m


def _nd_observed(n_obs, true_params, seed_obs, cov_matrix):
    simulator = partial(gauss_nd_mean, cov_matrix=cov_matrix, n_obs=n_obs)
    return simulator, simulator(*true_params, n_obs=n_obs,
                                random_state=np.random.RandomState(seed_obs))


def get_model(n_obs=50, true_params=None, seed_obs=None, nd_mean=False, cov_matrix=None):
    """elfi/examples/gauss.py:75-139: the 1-D model of mu and sigma, or with nd_mean=True the model
    of the D = len(true_params) means mu_0 .. mu_{D-1} (default [4, 4]) under cov_matrix (None:
    the identity)."""
    if nd_mean:
        if true_params is None:
            true_params = [4, 4]
        simulator, y_obs = _nd_observed(n_obs, true_params, seed_obs, cov_matrix)
        return _graph_nd(em.new_model(), [('uniform', t) for t in true_params], simulator, y_obs)
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


def gauss_nd_device(*mu, A, n_obs=15, batch_size=1, random_state=None):
    """Device twin of gauss_nd_mean for the factor A = ops.gauss_nd_factor(cov_matrix, D): a
    LazySimulation of shape (batch_size, n_obs, D) whose [means | variances] are computed in the
    simulator kernel; ``materialize()`` writes the data (once: later calls return the same
    tensor)."""
    cols = batch_columns(mu, batch_size)
    key = batch_key(random_state)
    data = []

    def materialize():
        if not data:
            data.append(ops.sim_gauss_nd(cols, A, n_obs, seed=key, want_data=True,
                                         want_summaries=False)[0])
        return data[0]

    return LazySimulation((int(cols[0].shape[0]), n_obs, len(cols)),
                          lambda kind: ops.sim_gauss_nd(cols, A, n_obs, seed=key)[1], materialize)


def get_device_model(n_obs=50, true_params=None, seed_obs=None, nd_mean=False, cov_matrix=None):
    """Gaussian noise inference task with priors, simulator and summaries on the device.

    Without nd_mean: returns (model, DeviceProposal instance).  With nd_mean=True: the n-D mean task
    of get_model(nd_mean=True) with the uniform priors drawn on the device (DeviceModelPrior), the
    device simulator with its summaries fused and the distance on the device; the observed data
    comes from the host simulator.  Returns (model, DeviceModelPrior); pass the latter as
    ``device_proposal=`` to SMC.  1 <= D <= ops.GAUSS_ND_D_MAX."""
    if nd_mean:
        if true_params is None:
            true_params = [4, 4]
        D = len(true_params)
        if not 1 <= D <= ops.GAUSS_ND_D_MAX:
            raise ValueError('the device n-D Gaussian model takes 1 <= D <= {} means, got {}'.format(
                ops.GAUSS_ND_D_MAX, D))
        if int(n_obs) != n_obs or not 1 <= n_obs <= ops.GAUSS_ND_NOBS_MAX:
            raise ValueError('the device n-D Gaussian simulator takes an integer 1 <= n_obs <= {}, '
                             'got {}'.format(ops.GAUSS_ND_NOBS_MAX, n_obs))
        A = ops.gauss_nd_factor(cov_matrix, D)
        _, y_obs = _nd_observed(n_obs, true_params, seed_obs, cov_matrix)
        m = _graph_nd(em.new_model(), [('uniform', t) for t in true_params],
                      partial(gauss_nd_device, A=A, n_obs=int(n_obs)), y_obs)
        dp = DeviceModelPrior(m)
        return dp.model, dp
    if true_params is None:
        true_params = [4, .4]
    y_obs = gauss(*true_params, n_obs=n_obs, random_state=np.random.RandomState(seed_obs))
    prm = _prior_params(true_params)
    m = _graph(em.new_model(), _DeviceUniform, _DeviceTruncnorm, prm,
               partial(gauss_device, n_obs=n_obs), y_obs)
    return m, DeviceProposal(prm)
