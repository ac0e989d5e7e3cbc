"""Bivariate g-and-k model (mirror of elfi/examples/bignk.py): nine parameters, the robust summary
ss_robust and the discrepancy euclidean_multiss of the univariate example (gnk.py).

The host path (BiGNK, get_model) consumes the batch's RandomState exactly as the reference does,
so it reproduces the reference's draws.  get_device_model is the same task in throughput mode:
stock uniform priors drawn on the device (DeviceModelPrior) and the simulator with its summaries
fused on the device (Philox streams; statistical parity with the host path)."""
from functools import partial

import numpy as np
import scipy.stats as ss
import torch

from .. import model as em
from .. import ops
from ..priors import DeviceModelPrior
from ..throughput import batch_columns, batch_key
from .gnk import euclidean_multiss, lazy_gnk, ss_robust

PARAMETER_NAMES = ['a1', 'a2', 'b1', 'b2', 'g1', 'g2', 'k1', 'k2', 'rho']


def BiGNK(A1, A2, B1, B2, g1, g2, k1, k2, rho, c=.8, n_obs=150, batch_size=1, random_state=None):
    """Bivariate g-and-k draws through the quantile function (bignk.py:12-108); output shape
    (batch_size, n_obs, 2).  z of row i ~ N(0, [[1, rho_i], [rho_i, 1]]), drawn per row with
    scipy's multivariate_normal from random_state, as the reference does."""
    A = np.hstack((np.asanyarray(A1).reshape((-1, 1)), np.asanyarray(A2).reshape((-1, 1))))
    B = np.hstack((np.asanyarray(B1).reshape((-1, 1)), np.asanyarray(B2).reshape((-1, 1))))
    g = np.hstack((np.asanyarray(g1).reshape((-1, 1)), np.asanyarray(g2).reshape((-1, 1))))
    k = np.hstack((np.asanyarray(k1).reshape((-1, 1, 1)), np.asanyarray(k2).reshape((-1, 1, 1))))
    rho = np.asanyarray(rho).reshape((-1, 1))

    z = np.array([ss.multivariate_normal.rvs(cov=np.array([[1, float(rho[i, 0])],
                                                           [float(rho[i, 0]), 1]]),
                                             size=n_obs, random_state=random_state)
                  for i in range(batch_size)])

    # the reference's operations and order (bignk.py:92-107)
    gdotz = np.einsum('ik,ijk->ijk', g, z)
    term_exp = (1 - np.exp(-gdotz)) / (1 + np.exp(-gdotz))
    term_first = np.einsum('ik,ijk->ijk', B, (1 + c * (term_exp)))
    k = np.swapaxes(np.repeat(k, n_obs, axis=2), 1, 2)
    term_second = np.power(1 + np.power(z, 2), k)
    term_product = term_first * term_second * z
    return np.swapaxes(np.add(A, np.swapaxes(term_product, 1, 0)), 1, 0)


def _priors(m):
    """bignk.py:134-144: the priors of Drovandi & Pettitt (2011), in the reference's order."""
    eps = np.finfo(float).eps
    prm = [(0, 5)] * 4 + [(-5, 10)] * 2 + [(-.5, 5.5)] * 2 + [(-1 + eps, 2 - 2 * eps)]
    return [em.Prior('uniform', lo, w, model=m, name=n) for n, (lo, w) in zip(PARAMETER_NAMES, prm)]


def _observed(n_obs, true_params, seed):
    if true_params is None:
        true_params = [3, 4, 1, 0.5, 1, 2, .5, .4, 0.6]
    return BiGNK(*true_params, n_obs=n_obs, random_state=np.random.RandomState(seed))


def get_model(n_obs=150, true_params=None, seed=None):
    """The bivariate g-and-k task (bignk.py:111-159): ss_robust + euclidean_multiss."""
    m = em.new_model()
    priors = _priors(m)
    em.Simulator(partial(BiGNK, n_obs=n_obs), *priors, observed=_observed(n_obs, true_params, seed),
                 name='BiGNK')
    default_ss = em.Summary(ss_robust, m['BiGNK'], name='ss_robust')
    em.Discrepancy(euclidean_multiss, default_ss, name='d')
    return m


# ---------------------------------------------------------------------------- throughput mode
def bignk_device(A1, A2, B1, B2, g1, g2, k1, k2, rho, c=.8, n_obs=150, batch_size=1,
                 random_state=None):
    """Device twin of BiGNK (Philox streams, ops.sim_bignk) with ss_robust / ss_octile fused into
    the simulator; returns a LazySimulation of shape (batch_size, n_obs, 2)."""
    P = torch.stack(batch_columns((A1, A2, B1, B2, g1, g2, k1, k2, rho), batch_size), dim=1)
    key = batch_key(random_state)
    return lazy_gnk(
        (int(P.shape[0]), n_obs, 2),
        lambda kind: ops.sim_bignk(P, n_obs, seed=key, c=c, want_data=False, kind=kind)[1],
        lambda: ops.sim_bignk(P, n_obs, seed=key, c=c)[0])


def get_device_model(n_obs=150, true_params=None, seed=None):
    """The bivariate g-and-k task in throughput mode: the graph of get_model with the nine stock
    uniform priors drawn on the device and the simulator and ss_robust fused on the device
    (n_obs <= 2048; the data is only written for n_obs > 512).  The observed data and its
    summaries are computed on the host.  Returns (model, DeviceModelPrior); pass the latter as
    ``device_proposal=`` to SMC."""
    if not 1 <= n_obs <= ops.GNK_SERIES_MAX:
        raise ValueError('device g-and-k summaries take 1 <= n_obs <= {}, got {}'.format(
            ops.GNK_SERIES_MAX, n_obs))
    m = em.new_model()
    priors = _priors(m)
    em.Simulator(partial(bignk_device, n_obs=n_obs), *priors,
                 observed=_observed(n_obs, true_params, seed), name='BiGNK')
    s = em.Summary(ss_robust, m['BiGNK'], name='ss_robust')
    em.Discrepancy(euclidean_multiss, s, name='d')
    dp = DeviceModelPrior(m)
    return dp.model, dp
