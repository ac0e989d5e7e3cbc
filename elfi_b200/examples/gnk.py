"""Univariate g-and-k model (mirror of elfi/examples/gnk.py) + the 2-d order-statistic variant that
BASELINE config #5 needs (AdaptiveDistance over a (B, n_obs) summary matrix).

ss_robust, ss_octile and euclidean_multiss take host arrays (the reference's NumPy code), device
tensors (the kernels of gnkstats.cu) and the lazy output of the throughput-mode simulators (the
summaries are computed in the simulator kernel); all three forms give the same bits."""
from functools import partial

import numpy as np
import scipy.stats as ss

from .. import device as dev
from .. import model as em
from .. import ops
from ..throughput import LazySimulation, batch_columns, batch_key


def GNK(A, B, g, k, c=0.8, n_obs=50, batch_size=1, random_state=None):
    """Sample the g-and-k distribution through its quantile function (gnk.py:11-68);
    output shape (batch_size, n_obs, 1)."""
    A = np.asanyarray(A).reshape((-1, 1))
    B = np.asanyarray(B).reshape((-1, 1))
    g = np.asanyarray(g).reshape((-1, 1))
    k = np.asanyarray(k).reshape((-1, 1))
    z = ss.norm.rvs(size=(batch_size, n_obs), random_state=random_state)
    y = A + B * (1 + c * ((1 - np.exp(-g * z)) / (1 + np.exp(-g * z)))) * (1 + z**2)**k * z
    return y[:, :, np.newaxis]


def ss_order(y):
    """gnk.py:145-161, reproduced as is: np.sort over the LAST axis of (B, n_obs, 1), i.e. the
    identity (SURVEY.md section 8a, a2)."""
    return np.sort(dev.to_host(y))


def ss_sorted(y):
    """Order statistics per simulation, (B, n_obs): np.sort(y[:, :, 0], axis=1) on the device."""
    y = dev.to_host(y) if not dev.is_device_array(y) else y
    y2 = y[:, :, 0] if y.ndim == 3 else y
    return ops.rowsort(np.ascontiguousarray(y2) if isinstance(y2, np.ndarray) else y2.contiguous())


def euclidean_multiss(*simulated, observed):
    """gnk.py:115-142 over 3-d summaries (B, K, 1); device summaries give a device (B,) result."""
    if dev.is_device_array(simulated[0]):
        return ops.euclidean_multiss(simulated[0], observed[0])
    pts_sim = dev.to_host(simulated[0])
    pts_obs = dev.to_host(observed[0])
    d_ss_merged = np.sum((pts_sim - pts_obs)**2., axis=1)
    return np.sqrt(np.sum(d_ss_merged, axis=1))


def _lazy_summaries(y, kind):
    """(B, width * d, 1) summaries of lazy simulator output or device data; None for host data."""
    if isinstance(y, LazySimulation):
        return y.summaries(kind)[:, :, None]
    if dev.is_device_array(y):
        return ops.gnk_summaries(y, kind)[:, :, None]
    return None


def ss_robust(y):
    """Robust summary of Drovandi & Pettitt (2011), gnk.py:164-188: (B, 4 d, 1) for y (B, n_obs, d),
    [A_1..A_d, B_1..B_d, g_1..g_d, k_1..k_d]."""
    s = _lazy_summaries(y, 'ss_robust')
    if s is not None:
        return s
    ss = np.hstack((_get_ss_A(y), _get_ss_B(y), _get_ss_g(y), _get_ss_k(y)))
    return ss[:, :, np.newaxis]


def ss_octile(y):
    """Octile summary, gnk.py:191-213: (B, 7 d, 1) for y (B, n_obs, d), [E1_1..E1_d, .., E7_d]."""
    s = _lazy_summaries(y, 'ss_octile')
    if s is not None:
        return s
    octiles = np.linspace(12.5, 87.5, 7)
    E1, E2, E3, E4, E5, E6, E7 = np.percentile(y, octiles, axis=1)
    return np.hstack((E1, E2, E3, E4, E5, E6, E7))[:, :, np.newaxis]


def _get_ss_A(y):
    """gnk.py:216-219: the median."""
    return np.percentile(y, 50, axis=1)


def _get_ss_B(y):
    """gnk.py:222-234: the interquartile range, eps where it is 0 (it divides ss_g and ss_k)."""
    L1, L3 = np.percentile(y, [25, 75], axis=1)
    ss_B = (L3 - L1).ravel()
    idxs_zero = np.where(ss_B == 0)[0]
    ss_B[idxs_zero] += np.finfo(float).eps
    return ss_B.reshape(y.shape[0], y.shape[-1])


def _get_ss_g(y):
    """gnk.py:237-241: skewness."""
    L1, L2, L3 = np.percentile(y, [25, 50, 75], axis=1)
    return np.divide(L3 + L1 - 2 * L2, _get_ss_B(y))


def _get_ss_k(y):
    """gnk.py:244-248: kurtosis."""
    E1, E3, E5, E7 = np.percentile(y, [12.5, 37.5, 62.5, 87.5], axis=1)
    return np.divide(E7 - E5 + E3 - E1, _get_ss_B(y))


def _base(n_obs, true_params, seed):
    m = em.new_model()
    if true_params is None:
        true_params = [3, 1, 2, .5]
    priors = [em.Prior('uniform', 0, 10, model=m, name=n) for n in ('A', 'B', 'g', 'k')]
    y_obs = GNK(*true_params, n_obs=n_obs, random_state=np.random.RandomState(seed))
    em.Simulator(partial(GNK, n_obs=n_obs), *priors, observed=y_obs, name='GNK')
    return m


def get_model(n_obs=50, true_params=None, seed=None):
    """Stock g-and-k task (gnk.py:71-112): ss_order + euclidean_multiss."""
    m = _base(n_obs, true_params, seed)
    default_ss = em.Summary(ss_order, m['GNK'], name='ss_order')
    em.Discrepancy(euclidean_multiss, default_ss, name='d')
    return m


def get_adaptive_model(n_obs=256, true_params=None, seed=None):
    """Config #5: (B, n_obs) order statistics + AdaptiveDistance (for AdaptiveDistanceSMC)."""
    m = _base(n_obs, true_params, seed)
    s = em.Summary(ss_sorted, m['GNK'], name='ss_sorted')
    em.AdaptiveDistance(s, name='d')
    return m


# ---------------------------------------------------------------------------- throughput mode
# Device-side priors, simulator and proposals (Philox streams; statistical parity with the host
# path).  The simulated (B, n_obs) matrix is born in HBM, sorted per row there (order statistics)
# and consumed by the nested-distance kernel; only accepted particles leave the device.
def gnk_device(A, B, g, k, c=0.8, n_obs=50, batch_size=1, random_state=None):
    """Device twin of GNK: returns a (batch_size, n_obs) CUDA tensor."""
    return ops.sim_gnk(*batch_columns((A, B, g, k), batch_size), n_obs=n_obs,
                       seed=batch_key(random_state), c=c)


class DeviceProposal:
    """SMC proposals / prior density on the device for the g-and-k model
    (pass an instance as ``device_proposal=`` to SMC / AdaptiveDistanceSMC)."""
    parameter_names = ['A', 'B', 'g', 'k']

    def __init__(self, lo=0.0, width=10.0):
        self.lo = np.broadcast_to(np.asarray(lo, dtype=np.float64), (4,)).copy()
        self.width = np.broadcast_to(np.asarray(width, dtype=np.float64), (4,)).copy()
        self.box = (list(self.lo), list(self.lo + self.width))

    def rvs(self, means, cov, weights, size, key, cdf=None):
        return ops.gm_rvs(means, cov, weights, size, seed=key, support=2, box=self.box, cdf=cdf)

    def logpdf(self, params):
        return ops.logprior_box(params, self.lo, self.width)


def lazy_gnk(shape, fused, materialize):
    """The LazySimulation of a g-and-k simulator of shape (B, n_obs, d): the robust / octile
    summaries of a kind are fused(kind) for n_obs <= ops.GNK_FUSED_MAX, else taken from the
    written data."""
    def summarise(kind):
        if shape[1] <= ops.GNK_FUSED_MAX:
            return fused(kind)
        return ops.gnk_summaries(materialize(), kind)
    return LazySimulation(shape, summarise, materialize)


def gnk_device_lazy(A, B, g, k, c=0.8, n_obs=50, batch_size=1, random_state=None):
    """Device twin of GNK whose robust / octile summaries are fused into the simulator; returns a
    LazySimulation of shape (batch_size, n_obs, 1)."""
    cols = batch_columns((A, B, g, k), batch_size)
    key = batch_key(random_state)
    return lazy_gnk(
        (int(cols[0].numel()), n_obs, 1),
        lambda kind: ops.sim_gnk_summaries(*cols, n_obs=n_obs, seed=key, c=c, kind=kind),
        lambda: ops.sim_gnk(*cols, n_obs=n_obs, seed=key, c=c)[:, :, None])


def get_device_model(n_obs=256, true_params=None, seed=None, summary='ss_sorted'):
    """The g-and-k task in throughput mode: uniform(0, 10) priors drawn on the device and the
    simulator on the device.  Returns (model, DeviceProposal).

    summary='ss_sorted': config #5, row-sorted order statistics and AdaptiveDistance.
    summary='ss_robust' or 'ss_octile': the reference's get_model graph with that summary and
    euclidean_multiss; the summaries are fused into the simulator (n_obs <= 2048; the data is
    only written for n_obs > 512).  The observed summaries are computed on the host."""
    from .gauss import _DeviceUniform
    if summary not in ('ss_sorted', 'ss_robust', 'ss_octile'):
        raise ValueError("summary must be 'ss_sorted', 'ss_robust' or 'ss_octile', got {!r}".format(
            summary))
    if summary != 'ss_sorted' and not 1 <= n_obs <= ops.GNK_SERIES_MAX:
        raise ValueError('device g-and-k summaries take 1 <= n_obs <= {}, got {}'.format(
            ops.GNK_SERIES_MAX, n_obs))
    if true_params is None:
        true_params = [3, 1, 2, .5]
    m = em.new_model()
    priors = [em.Prior(_DeviceUniform, 0, 10, model=m, name=n) for n in ('A', 'B', 'g', 'k')]
    y_obs = GNK(*true_params, n_obs=n_obs, random_state=np.random.RandomState(seed))
    if summary == 'ss_sorted':
        em.Simulator(partial(gnk_device, n_obs=n_obs), *priors, observed=y_obs, name='GNK')
        s = em.Summary(ss_sorted, m['GNK'], name='ss_sorted')
        em.AdaptiveDistance(s, name='d')
    else:
        em.Simulator(partial(gnk_device_lazy, n_obs=n_obs), *priors, observed=y_obs, name='GNK')
        s = em.Summary(ss_robust if summary == 'ss_robust' else ss_octile, m['GNK'], name=summary)
        em.Discrepancy(euclidean_multiss, s, name='d')
    return m, DeviceProposal()

