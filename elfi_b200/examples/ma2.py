"""MA2 model (mirror of elfi/examples/ma2.py) with device summaries.

The simulator and priors run on the host with the per-batch RandomState exactly as in the
reference (that is what "same seeds" means, SURVEY.md section 7); the summaries and the distance
run on the device.
"""
from functools import partial

import numpy as np
import scipy.stats as ss

from .. import model as em
from .. import ops
from ..throughput import LazySimulation, batch_columns, batch_key


def MA2(t1, t2, n_obs=100, batch_size=1, random_state=None):
    """x_i = w_i + t1 w_{i-1} + t2 w_{i-2}, w ~ N(0,1)  (elfi/examples/ma2.py:11-37)."""
    t1 = np.asanyarray(t1).reshape((-1, 1))
    t2 = np.asanyarray(t2).reshape((-1, 1))
    random_state = random_state or np.random
    w = random_state.randn(batch_size, n_obs + 2)
    x = w[:, 2:] + t1 * w[:, 1:-1] + t2 * w[:, :-2]
    return x


def autocov(x, lag=1):
    """Autocovariance summary on the device (elfi/examples/ma2.py:40-59); returns (B,).  Lags 1 and
    2 of lazy simulator output come from the simulator kernel, other lags from its data."""
    if isinstance(x, LazySimulation):
        if lag in (1, 2):
            return x.summaries()[:, lag - 1]
        x = x.materialize()
    x = np.atleast_2d(x) if not hasattr(x, 'is_cuda') else x
    return ops.autocov(x, lags=(lag,))[:, 0]


class CustomPrior1:
    """Triangular prior of t1 on [-b, b] (elfi/examples/ma2.py:96-140)."""

    @classmethod
    def rvs(cls, b, size=1, random_state=None):
        u = ss.uniform.rvs(loc=0, scale=1, size=size, random_state=random_state)
        return np.where(u < 0.5, np.sqrt(2. * u) * b - b, -np.sqrt(2. * (1. - u)) * b + b)

    @classmethod
    def pdf(cls, x, b):
        p = 1. / b - np.abs(x) / (b * b)
        return np.where(p < 0., 0., p)

    @classmethod
    def logpdf(cls, x, b):
        with np.errstate(divide='ignore'):
            return np.log(cls.pdf(x, b))


class CustomPrior2:
    """Uniform prior of t2 given t1 (elfi/examples/ma2.py:143-186)."""

    @classmethod
    def rvs(cls, t1, a, size=1, random_state=None):
        locs = np.maximum(-a - t1, -a + t1)
        scales = a - locs
        return ss.uniform.rvs(loc=locs, scale=scales, size=size, random_state=random_state)

    @classmethod
    def pdf(cls, x, t1, a):
        locs = np.maximum(-a - t1, -a + t1)
        scales = a - locs
        return (x >= locs) * (x <= locs + scales) * 1 / np.where(scales > 0, scales, 1)

    @classmethod
    def logpdf(cls, x, t1, a):
        with np.errstate(divide='ignore'):
            return np.log(cls.pdf(x, t1, a))


def _graph(m, prior1, prior2, simulator, y):
    """Priors, simulator, summaries and distance of elfi/examples/ma2.py:62-92."""
    em.Prior(prior1, 2, model=m, name='t1')
    em.Prior(prior2, m['t1'], 1, name='t2')
    em.Simulator(simulator, m['t1'], m['t2'], observed=y, name='MA2')
    em.Summary(autocov, m['MA2'], name='S1')
    em.Summary(autocov, m['MA2'], 2, name='S2')
    em.Distance('euclidean', m['S1'], m['S2'], name='d')
    return m


def _observed(n_obs, true_params, seed_obs):
    if true_params is None:
        true_params = [.6, .2]
    return MA2(*true_params, n_obs=n_obs, random_state=np.random.RandomState(seed_obs))


def get_model(n_obs=100, true_params=None, seed_obs=None):
    """MA2 inference task (elfi/examples/ma2.py:62-92)."""
    return _graph(em.ElfiModel(), CustomPrior1, CustomPrior2, partial(MA2, n_obs=n_obs),
                  _observed(n_obs, true_params, seed_obs))


# ---------------------------------------------------------------------------- throughput mode
# Everything below keeps a batch on the device from the prior draw to the distance: priors,
# simulator and summaries use counter-based Philox streams (statistically equivalent to the
# host RandomState of the reference, not bit-identical; SURVEY.md section 7 "Philox throughput
# mode").  The per-node key is drawn from the batch's host RandomState, so results stay a
# deterministic function of (seed, batch_index).
def MA2_device(t1, t2, n_obs=100, batch_size=1, random_state=None):
    """Device twin of MA2 with autocov lags 1 and 2 fused into the simulator; returns a
    LazySimulation."""
    t1, t2 = batch_columns((t1, t2), batch_size)
    key = batch_key(random_state)
    return LazySimulation(
        (int(t1.numel()), n_obs),
        lambda kind: ops.sim_ma2(t1, t2, n_obs, seed=key)[1],
        lambda: ops.sim_ma2(t1, t2, n_obs, seed=key, want_data=True, want_summaries=False)[0])


class DevicePrior1(CustomPrior1):
    @classmethod
    def rvs(cls, b, size=1, random_state=None):
        assert b == 2, 'device MA2 prior is specialised to b = 2'
        n = int(np.prod(size))
        return ops.prior_ma2(n, batch_key(random_state), which='t1')


class DevicePrior2(CustomPrior2):
    @classmethod
    def rvs(cls, t1, a, size=1, random_state=None):
        assert a == 1, 'device MA2 prior is specialised to a = 1'
        return ops.prior_ma2(0, batch_key(random_state), t1=t1, which='t2')


class DeviceProposal:
    """Device replacements of the two host-side pieces of SMC.prepare_new_batch /
    _compute_weights (samplers.py:434-459, 512): proposal draws restricted to the prior support
    and the joint prior log density."""
    parameter_names = ['t1', 't2']

    @staticmethod
    def rvs(means, cov, weights, size, key, cdf=None):
        return ops.gm_rvs(means, cov, weights, size, seed=key, support=1, cdf=cdf)

    @staticmethod
    def logpdf(params):
        return ops.logprior_ma2(params)


def get_device_model(n_obs=100, true_params=None, seed_obs=None):
    """MA2 inference task with priors, simulator and summaries on the device (same graph and
    names as get_model).  Pass ``device_proposal=DeviceProposal`` to SMC for device proposals."""
    return _graph(em.ElfiModel(), DevicePrior1, DevicePrior2, partial(MA2_device, n_obs=n_obs),
                  _observed(n_obs, true_params, seed_obs))


def get_uniform_device_model(n_obs=100, true_params=None, seed_obs=None):
    """MA2 in throughput mode with stock uniform priors, t1 ~ U(-2, 2) and t2 ~ U(-1, 1) (the box
    around the reference's triangular prior, which the device prior table does not cover), drawn
    on the device, and the device simulator and summaries.  Returns (model, DeviceModelPrior);
    pass the latter as ``device_proposal=`` to SMC or BSL."""
    from ..priors import DeviceModelPrior
    m = em.ElfiModel()
    em.Prior('uniform', -2, 4, model=m, name='t1')
    em.Prior('uniform', -1, 2, model=m, name='t2')
    em.Simulator(partial(MA2_device, n_obs=n_obs), m['t1'], m['t2'],
                 observed=_observed(n_obs, true_params, seed_obs), name='MA2')
    em.Summary(autocov, m['MA2'], name='S1')
    em.Summary(autocov, m['MA2'], 2, name='S2')
    em.Distance('euclidean', m['S1'], m['S2'], name='d')
    dp = DeviceModelPrior(m)
    return dp.model, dp
