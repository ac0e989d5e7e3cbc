"""Alpha-stable stochastic volatility model (mirror of
elfi/examples/stochastic_volatility_model.py; Vankov et al. 2019, Priddle and Drovandi 2020): returns
y_t = exp(x_t / 2) v_t with an AR(1) log-volatility x_t (mean mu, persistence phi, noise scale
sigma) and alpha-stable shocks v_t ~ S0(alpha, beta, kappa, eta), summarised by a quantile kurtosis
and skewness.

alpha and beta are inferred; kappa, eta, mu, phi and sigma are Constant nodes, parents of the
simulator as in the reference.

The host path (alpha_stochastic_volatility_model, shock_term, log_vol, kurt, skew, get_model)
consumes the batch's RandomState exactly as the reference does, so it reproduces the reference's
draws.  get_device_model is the same task in throughput mode: the uniform priors drawn on the device
(DeviceModelPrior), the simulator with both summaries fused on the device (Philox streams;
statistical parity with the host path).

kurt and skew take host arrays (the reference's NumPy code), device tensors (ops.row_quantiles, then
the same fp64 arithmetic in torch) and the lazy output of the device simulator (the summaries
computed in the simulator); all forms give the same bits."""
import logging
from functools import partial

import numpy as np
import scipy.stats as ss
import torch

from .. import device as dev
from .. import model as em
from .. import ops
from ..priors import DeviceModelPrior
from ..throughput import LazySimulation, batch_columns, batch_key

logger = logging.getLogger(__name__)

FIXED = {'kappa': 1, 'eta': 0, 'mu': 0, 'phi': 0.95, 'sigma': 0.2}


def shock_term(alpha, beta, kappa, eta, n_obs, batch_size=1, random_state=None):
    """levy_stable(alpha, beta, loc=eta, scale=kappa) draws of shape (n_obs, batch_size) in the S0
    parameterization, set on the frozen distribution's own instance as the reference does."""
    distribution = ss.levy_stable(alpha=alpha, beta=beta, loc=eta, scale=kappa)
    distribution.dist.parameterization = 'S0'
    distribution.random_state = random_state
    return distribution.rvs(size=(n_obs, batch_size))


def log_vol(mu, phi, sigma, n_obs, prev_x=None, batch_size=1, random_state=None):
    """The AR(1) log-volatility (n_obs, batch_size), drawn t-major with norm.rvs: x_0 from the
    stationary N(mu, sigma / sqrt(1 - min(phi^2, 0.99999))), or from prev_x by the recurrence;
    x_t ~ N(mu + phi (x_{t-1} - mu), sigma)."""
    x = np.zeros((n_obs, batch_size))
    if prev_x is None:
        scale = sigma / np.sqrt((1 - np.minimum(np.squeeze(phi) ** 2, 0.99999)))
        x[0] = ss.norm.rvs(mu, scale, batch_size, random_state=random_state)
    else:
        x[0] = ss.norm.rvs(mu + phi * (prev_x - mu), sigma, batch_size, random_state=random_state)
    for t in range(1, n_obs):
        x[t] = ss.norm.rvs(mu + phi * (x[t - 1] - mu), sigma, batch_size,
                           random_state=random_state)
    return x


def alpha_stochastic_volatility_model(alpha, beta, kappa, eta, mu, phi, sigma, n_obs=50, x_0=None,
                                      batch_size=1, random_state=None):
    """(batch_size, n_obs) returns exp(0.5 x) * v: the log-volatility is drawn first, then the
    shocks."""
    x_t = log_vol(mu, phi, sigma, n_obs, x_0, batch_size, random_state)
    v_t = shock_term(alpha, beta, kappa, eta, n_obs, batch_size, random_state)
    return np.transpose(np.exp(0.5 * x_t) * v_t)


def _device_summaries(x):
    """[kurt, skew] (B, 2) of lazy simulator output or device data; None for host data."""
    if isinstance(x, LazySimulation):
        return x.summaries()
    if dev.is_device_array(x):
        return ops.svm_summaries(x)
    return None


def kurt(x):
    """(q95 - q05) / (q75 - q25) of each row's np.quantile, (batch_size,)."""
    s = _device_summaries(x)
    if s is not None:
        return s[:, 0]
    qs = np.quantile(x, q=[0.05, 0.25, 0.75, 0.95], axis=1)
    return np.transpose((qs[3] - qs[0]) / (qs[2] - qs[1]))


def skew(x):
    """((q95 - q50) - (q50 - q05)) / (q95 - q05) of each row's np.quantile, (batch_size,)."""
    s = _device_summaries(x)
    if s is not None:
        return s[:, 1]
    qs = np.quantile(x, q=[0.05, 0.50, 0.95], axis=1)
    return np.transpose((((qs[2] - qs[1]) - (qs[1] - qs[0])) / (qs[2] - qs[0])))


def _graph(m, simulator, y_obs):
    """Priors, Constants, simulator, summaries and distance of the reference's get_model."""
    em.Prior('uniform', 0.5, 1.5, model=m, name='alpha')
    em.Prior('uniform', -1, 2, model=m, name='beta')
    constants = [em.Constant(value, model=m, name=name) for name, value in FIXED.items()]
    em.Simulator(simulator, m['alpha'], m['beta'], *constants, observed=y_obs, name='a_svm')
    em.Summary(kurt, m['a_svm'], name='kurt')
    em.Summary(skew, m['a_svm'], name='skew')
    em.Distance('euclidean', m['kurt'], m['skew'], name='d')
    return m


def _observed(n_obs, true_params, seed_obs):
    if true_params is None:
        true_params = [1.2, 0.5]
    y = alpha_stochastic_volatility_model(*true_params, **FIXED, n_obs=n_obs,
                                          random_state=np.random.RandomState(seed_obs))
    logger.info("Generated observations with true parameters alpha: %.1f, beta: %.1f",
                *true_params)
    return y


def get_model(n_obs=50, true_params=None, seed_obs=None):
    """The stochastic volatility task: priors alpha ~ U(0.5, 2), beta ~ U(-1, 1), the Constants
    kappa = 1, eta = 0, mu = 0, phi = 0.95, sigma = 0.2, the simulator 'a_svm', the summaries
    'kurt' and 'skew' and their Euclidean distance 'd'."""
    y_obs = _observed(n_obs, true_params, seed_obs)
    simulator = partial(alpha_stochastic_volatility_model, n_obs=n_obs)
    return _graph(em.new_model(), simulator, y_obs)


# ---------------------------------------------------------------------------- throughput mode
def svm_device(alpha, beta, kappa, eta, mu, phi, sigma, n_obs=50, x_0=None, batch_size=1,
               random_state=None):
    """Device twin of alpha_stochastic_volatility_model: a LazySimulation of shape (batch_size,
    n_obs) whose [kurt, skew] are computed in the simulator kernel.  The log-volatility starts from
    its stationary law; x_0 is not supported on the device."""
    if x_0 is not None:
        raise ValueError('x_0 is not supported by the device stochastic volatility simulator; use '
                         'alpha_stochastic_volatility_model')
    P = torch.stack(batch_columns((alpha, beta, kappa, eta, mu, phi, sigma), batch_size), dim=1)
    key = batch_key(random_state)
    return LazySimulation(
        (int(P.shape[0]), n_obs),
        lambda kind: ops.sim_svm(P, n_obs, seed=key)[1],
        lambda: ops.sim_svm(P, n_obs, seed=key, want_data=True, want_summaries=False)[0])


def get_device_model(n_obs=50, true_params=None, seed_obs=None):
    """The stochastic volatility task in throughput mode: the graph of get_model (the Constants
    parents of the simulator) with the uniform priors drawn on the device and the device simulator
    with kurt and skew fused into it.  The observed data and its summaries are computed on the
    host.  Returns (model, DeviceModelPrior); pass the latter as ``device_proposal=`` to SMC."""
    ops._mg1_n(n_obs, 'the device stochastic volatility simulator and its summaries')
    y_obs = _observed(n_obs, true_params, seed_obs)
    m = _graph(em.new_model(), partial(svm_device, n_obs=n_obs), y_obs)
    dp = DeviceModelPrior(m)
    return dp.model, dp
