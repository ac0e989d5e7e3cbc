"""M/G/1 queue model (mirror of elfi/examples/mg1.py): customers arrive with Exp(t3) inter-arrival
times and are served in U(t1, t2) time; the data are the n_obs inter-departure times, summarised by
their log (An et al. 2020) and by equidistant quantiles (Blum and Francois 2010).

The prior is hierarchical: t2 ~ U(t1, t1 + 10), a uniform whose loc is the prior t1.

The host path (MG1, log_identity, quantiles, get_model) consumes the batch's RandomState exactly as
the reference does, so it reproduces the reference's draws.  get_device_model is the same task in
throughput mode: the priors drawn on the device (DeviceModelPrior with conditional=True, which
takes t2's loc from t1 per row), the simulator with its quantiles fused on the device (Philox
streams; statistical parity with the host path).

quantiles takes host arrays (the reference's NumPy code), device tensors (ops.row_quantiles) and
the lazy output of the device simulator (the quantiles computed in the simulator); all forms give
the same bits.  log_identity of device data is torch.log of the materialised data, within an ulp or
two of np.log, not bit-equal to it."""
import logging
from functools import partial

import numpy as np
import torch

from .. import device as dev
from .. import model as em
from .. import ops
from ..priors import DeviceModelPrior
from ..throughput import LazySimulation, batch_columns, batch_key

logger = logging.getLogger(__name__)


def MG1(t1, t2, t3, n_obs=50, batch_size=1, random_state=None):
    """Inter-departure times of the M/G/1 queue (mg1.py:21-54): W ~ Exp(t3) arrival gaps and
    U ~ U(t1, t2) service times, all W (n_obs, batch_size) drawn first, then all U; returns
    (batch_size, n_obs)."""
    random_state = random_state or np.random
    W = random_state.exponential(1 / t3, size=(n_obs, batch_size))
    U = random_state.uniform(t1, t2, size=(n_obs, batch_size))
    y = np.zeros((n_obs, batch_size))
    sum_w = np.zeros(batch_size)
    sum_x = np.zeros(batch_size)
    for i in range(n_obs):
        sum_w += W[i]
        y[i] = U[i] + np.maximum(0, sum_w - sum_x)
        sum_x += y[i]
    return np.transpose(y)


def log_identity(x):
    """np.log(x), the summary 'log_identity' (mg1.py:57-59); torch.log of the data on the device."""
    if isinstance(x, LazySimulation):
        x = x.materialize()
    if dev.is_device_array(x):
        return torch.log(x)
    return np.log(x)


def quantiles(x, q):
    """np.quantile(x, q, axis=1).T, the summary 'quantiles' (mg1.py:62-65)."""
    if isinstance(x, LazySimulation):
        if np.array_equal(np.asarray(q, dtype=np.float64).reshape(-1), x.q):
            return x.summaries()
        x = x.materialize()
    if dev.is_device_array(x):
        return ops.row_quantiles(x, q)
    qs = np.quantile(x, q, axis=1)
    return np.transpose(qs)


def _graph(m, simulator, y_obs, n_quantiles):
    """Priors, simulator, summaries and distance of mg1.py:96-114."""
    em.Prior('uniform', 0, 10, model=m, name='t1')
    em.Prior('uniform', m['t1'], 10, model=m, name='t2')      # t2 - t1 ~ U(0, 10)
    em.Prior('uniform', 0, 0.5, model=m, name='t3')
    em.Simulator(simulator, m['t1'], m['t2'], m['t3'], observed=y_obs, name='MG1')
    em.Summary(log_identity, m['MG1'], name='log_identity')
    q = np.linspace(0, 1, n_quantiles)
    em.Summary(partial(quantiles, q=q), m['MG1'], name='quantiles')
    em.Distance('euclidean', m['quantiles'], w=(1 / 100) ** q, name='d')
    return m


def _observed(n_obs, true_params, seed_obs):
    if true_params is None:
        true_params = [1., 5., 0.2]
    y = MG1(*true_params, n_obs=n_obs, random_state=np.random.RandomState(seed_obs))
    logger.info("Generated observations with true parameters t1: %.1f, t2: %.1f, t3: %.1f, ",
                *true_params)
    return y


def get_model(n_obs=50, true_params=None, seed_obs=None, n_quantiles=10):
    """The M/G/1 inference task of mg1.py:68-116: priors t1 ~ U(0, 10), t2 ~ U(t1, t1 + 10),
    t3 ~ U(0, 0.5), the simulator 'MG1', the summaries 'log_identity' and 'quantiles' (n_quantiles
    equidistant levels) and the weighted Euclidean distance 'd' on the quantiles, w = 100^-q."""
    y_obs = _observed(n_obs, true_params, seed_obs)
    return _graph(em.new_model(), partial(MG1, n_obs=n_obs), y_obs, n_quantiles)


# ---------------------------------------------------------------------------- throughput mode
def mg1_device(t1, t2, t3, n_obs=50, q=np.linspace(0, 1, 10), batch_size=1, random_state=None):
    """Device twin of MG1: a LazySimulation of shape (batch_size, n_obs) whose quantiles at q are
    computed in the simulator kernel."""
    P = torch.stack(batch_columns((t1, t2, t3), batch_size), dim=1)
    key = batch_key(random_state)
    qv = np.asarray(q, dtype=np.float64).reshape(-1)
    lazy = LazySimulation(
        (int(P.shape[0]), n_obs),
        lambda kind: ops.sim_mg1(P, n_obs, qv, seed=key)[1],
        lambda: ops.sim_mg1(P, n_obs, qv, seed=key, want_data=True, want_summaries=False)[0])
    lazy.q = qv
    return lazy


def get_device_model(n_obs=50, true_params=None, seed_obs=None, n_quantiles=10):
    """The M/G/1 task in throughput mode: the graph of get_model with the priors drawn on the device
    (t2's loc taken from t1 per row) and the device simulator with its quantiles fused into it.  The
    observed data and its summaries are computed on the host.  Returns (model, DeviceModelPrior);
    pass the latter as ``device_proposal=`` to SMC."""
    ops._mg1_n(n_obs, 'the device M/G/1 simulator and its quantiles')
    q = np.linspace(0, 1, n_quantiles)
    ops._mg1_q(q)
    y_obs = _observed(n_obs, true_params, seed_obs)
    m = _graph(em.new_model(), partial(mg1_device, n_obs=n_obs, q=q), y_obs, n_quantiles)
    dp = DeviceModelPrior(m, conditional=True)
    return dp.model, dp
