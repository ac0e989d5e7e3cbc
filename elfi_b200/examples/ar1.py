"""AR(1) model (mirror of elfi/examples/ar1.py): x_t = phi x_{t-1} + w_t with white noise
w_t ~ N(0, 1) and x_0 = 0, compared with the observed series by the Euclidean distance of the raw
series (there are no summaries).

The host path (AR1, get_model) consumes the batch's RandomState exactly as the reference does, so
it reproduces the reference's draws.  get_device_model is the same task in throughput mode: the
uniform prior drawn on the device (DeviceModelPrior) and the device simulator, whose Euclidean
distance to the observed series is computed in the simulator kernel, so a batch writes one double
per row instead of its n_obs observations (Philox streams; statistical parity with the host path).
"""
import logging
from functools import partial

import numpy as np

from .. import model as em
from .. import ops
from ..priors import DeviceModelPrior
from ..throughput import LazySimulation, batch_columns, batch_key

logger = logging.getLogger(__name__)


def AR1(phi, n_obs=200, batch_size=1, random_state=None):
    """The AR(1) series (ar1.py:11-38): (batch_size, n_obs) rows x_1 .. x_n.  The innovations are
    drawn as one (batch_size, n_obs + 1) block whose column 0 is never used, as in the
    reference."""
    phi = np.asanyarray(phi)
    random_state = random_state or np.random
    w = random_state.randn(batch_size, n_obs + 1)
    x = np.zeros((batch_size, n_obs))
    prev = np.zeros(batch_size)
    for t in range(n_obs):
        x[:, t] = phi * prev + w[:, t + 1]
        prev = x[:, t]
    return x


def _graph(m, simulator, y_obs):
    """Prior, simulator and distance of ar1.py:63-68."""
    em.Prior('uniform', -1, 2, model=m, name='phi')
    em.Simulator(simulator, m['phi'], observed=y_obs, name='AR1')
    em.Distance('euclidean', m['AR1'], name='d')
    return m


def _observed(n_obs, true_params, seed_obs):
    if true_params is None:
        true_params = [.9]
    y = AR1(*true_params, n_obs=n_obs, random_state=np.random.RandomState(seed_obs))
    logger.info('Generated observations with true parameter phi: %.1f.', *true_params)
    return y


def get_model(n_obs=200, true_params=None, seed_obs=None):
    """The AR(1) inference task of ar1.py:41-72: the uniform prior phi on [-1, 1], the simulator
    'AR1' and the Euclidean distance 'd' of the simulated series to the observed one."""
    return _graph(em.new_model(), partial(AR1, n_obs=n_obs), _observed(n_obs, true_params, seed_obs))


# ---------------------------------------------------------------------------- throughput mode
def ar1_device(phi, n_obs=200, batch_size=1, random_state=None):
    """Device twin of AR1: a LazySimulation of shape (batch_size, n_obs).  Its Euclidean distance
    to an observed series is computed in the simulator kernel; ``materialize()`` writes the series
    (once: later calls return the same tensor).  It has no fused summaries."""
    phi_col, = batch_columns((phi,), batch_size)
    key = batch_key(random_state)
    data = []

    def materialize():
        if not data:
            data.append(ops.sim_ar1(phi_col, n_obs, seed=key, want_data=True)[0])
        return data[0]

    def summarise(kind):
        raise ValueError('the AR(1) simulator has no fused summaries: call materialize() on its '
                         'output and summarise the series')

    def euclidean(obs, thresholds):
        return ops.sim_ar1(phi_col, n_obs, seed=key, obs=obs, thresholds=thresholds,
                           want_data=False)[1:]

    return LazySimulation((int(phi_col.shape[0]), n_obs), summarise, materialize,
                          euclidean=euclidean)


def get_device_model(n_obs=200, true_params=None, seed_obs=None):
    """The AR(1) task in throughput mode: the graph of get_model with the uniform prior drawn on
    the device and the device simulator with the distance fused into it.  The observed series is
    computed on the host, as in get_model.  Returns (model, DeviceModelPrior); pass the latter as
    ``device_proposal=`` to SMC."""
    if int(n_obs) != n_obs or not 1 <= n_obs <= ops.AR1_NOBS_MAX:
        raise ValueError('the device AR(1) simulator takes an integer 1 <= n_obs <= {}, got '
                         '{}'.format(ops.AR1_NOBS_MAX, n_obs))
    y_obs = _observed(n_obs, true_params, seed_obs)
    m = _graph(em.new_model(), partial(ar1_device, n_obs=int(n_obs)), y_obs)
    dp = DeviceModelPrior(m)
    return dp.model, dp
