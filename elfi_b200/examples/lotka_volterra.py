"""Stochastic Lotka-Volterra predator-prey model (mirror of elfi/examples/lotka_volterra.py; Owen,
Wilkinson & Gillespie 2015): a Markov jump process with the reactions prey -> 2 prey (rate r1 X),
prey + predator -> 2 predators (rate r2 X Y) and predator -> 0 (rate r3 Y), simulated by Gillespie's
direct method and observed at n_obs evenly spaced times, optionally with Gaussian noise.  Nine
summaries: the means, log variances and lag-1 and lag-2 autocorrelations of both species, and their
cross-correlation.

The host path (lotka_volterra, the summaries, get_model) consumes the batch's RandomState exactly as
the reference does, so it reproduces the reference's draws.  get_device_model is the same task in
throughput mode: the priors drawn on the device, the simulator on the device (one lane per row,
lanes refilled with new rows as theirs finish; Philox streams, statistical parity with the host
path) and the nine summaries in one kernel.

The summaries take host arrays (the reference's NumPy code), device tensors (ops.lv_summaries) and
the lazy output of the device simulator; all forms give the same values, except that the device's
log may differ from NumPy's by an ulp."""
from functools import partial

import numpy as np
import scipy.stats as ss
import torch

from .. import device as dev
from .. import model as em
from .. import ops
from ..priors import DevicePriorDistribution, prior_spec
from ..throughput import LazySimulation, batch_columns, batch_key

N_FULL = 20000          # events per row kept before the event arrays are doubled
# the change of (prey, predators) of reactions R1, R2, R3 and of the null reaction
STOICHIOMETRY = np.array([[1, 0], [-1, 1], [0, -1], [0, 0]], dtype=np.int32)
SUMMARY_NAMES = ('prey_mean', 'pred_mean', 'prey_log_var', 'pred_log_var', 'prey_autocorr_1',
                 'pred_autocorr_1', 'prey_autocorr_2', 'pred_autocorr_2', 'crosscorr')


def lotka_volterra(r1, r2, r3, prey_init=50, predator_init=100, sigma=0., n_obs=16, time_end=30.,
                   batch_size=1, random_state=None, return_full=False):
    """The Lotka-Volterra simulator (lotka_volterra.py:18-143): (batch_size, n_obs, 2) int32 counts
    of prey and predators at np.linspace(0, time_end, n_obs).

    The whole batch steps together until every row has reached time_end.  A step draws
    exponential(1 / total hazard) (batch_size) for the waiting times, then uniform (batch_size, 1)
    for the reactions; a total hazard of 0 gives an infinite time and the null reaction, and an
    event that leaves no predators gets the time time_end.  Observation j >= 1 interpolates linearly
    between the last event before its time and the first at or after it, adds normal(scale=sigma)
    (batch_size) noise to the prey and then to the predators, and truncates toward zero.  With
    return_full the result is (observations, observation times, every event's counts, event times);
    beyond 20000 steps the counts are float64."""
    random_state = random_state or np.random
    r1, r2, r3, prey_init, predator_init, sigma = (
        np.asanyarray(v).reshape(-1) for v in (r1, r2, r3, prey_init, predator_init, sigma))

    cap = N_FULL
    stock = np.empty((batch_size, cap, 2), dtype=np.int32)
    # the continuous priors of the initial counts are rounded down
    stock[:, 0, 0] = np.floor(prey_init)
    stock[:, 0, 1] = np.floor(predator_init)
    times = np.empty((batch_size, cap))
    times[:, 0] = 0

    k = 0
    while np.any(times[:, k] < time_end):
        k += 1
        if k == cap:
            # np.empty is float64: from here on the counts are float64
            stock = np.concatenate((stock, np.empty((batch_size, cap, 2))), axis=1)
            times = np.concatenate((times, np.empty((batch_size, cap))), axis=1)
            cap *= 2
        prey, pred = stock[:, k - 1, 0], stock[:, k - 1, 1]
        hazards = np.column_stack((r1 * prey, r2 * prey * pred, r3 * pred))
        with np.errstate(divide='ignore', invalid='ignore'):
            inv_total = 1. / np.sum(hazards, axis=1, keepdims=True)
            times[:, k] = times[:, k - 1] + random_state.exponential(inv_total.ravel())
            thresholds = np.cumsum((hazards * inv_total)[:, :-1], axis=1)
            u = random_state.uniform(size=(batch_size, 1))
            reaction = np.sum(u >= thresholds, axis=1)
        # the null reaction when nothing can happen (infinite time)
        reaction = np.where(np.isinf(inv_total.ravel()), 3, reaction)
        stock[:, k, :] = stock[:, k - 1, :] + STOICHIOMETRY[reaction, :]
        # nothing more to see once the predators are gone
        times[:, k] = np.where(stock[:, k, 1] == 0, time_end, times[:, k])

    stock = stock[:, :k + 1, :]
    times = times[:, :k + 1]

    times_out = np.linspace(0, time_end, n_obs)
    stock_out = np.empty((batch_size, n_obs, 2), dtype=np.int32)
    stock_out[:, 0, :] = stock[:, 0, :]
    for j in range(1, n_obs):
        rows, cols = np.where(times >= times_out[j])
        rows, first = np.unique(rows, return_index=True)
        before = cols[first] - 1
        frac = (times_out[j] - times[rows, before]) / (times[rows, before + 1] - times[rows, before])
        for s in (0, 1):
            stock_out[:, j, s] = (stock[rows, before + 1, s] - stock[rows, before, s]) * frac \
                + stock[rows, before, s] + random_state.normal(scale=sigma, size=batch_size)

    if return_full:
        return stock_out, times_out, stock, times
    return stock_out


# ---------------------------------------------------------------------------- summaries
def _device_summaries(stock):
    """The (B, 9) summaries of lazy simulator output or device data; None for host data."""
    if isinstance(stock, LazySimulation):
        return stock.summaries()
    if dev.is_device_array(stock):
        return ops.lv_summaries(stock)
    return None


def _column(S, col, mu, std):
    c = S[:, col]
    return c if (mu == 0 and std == 1) else (c - mu) / std


def stock_mean(stock, species=0, mu=0, std=1):
    """The mean of a species' observations (lotka_volterra.py:226-231)."""
    S = _device_summaries(stock)
    if S is not None:
        return _column(S, species, mu, std)
    x = np.atleast_2d(stock[:, :, species])
    return (np.mean(x, axis=1) - mu) / std


def stock_log_variance(stock, species=0, mu=0, std=1):
    """log(var + 1) of a species' observations, var with ddof = 1 (lotka_volterra.py:234-240)."""
    S = _device_summaries(stock)
    if S is not None:
        return _column(S, 2 + species, mu, std)
    x = np.atleast_2d(stock[:, :, species])
    return (np.log(np.var(x, axis=1, ddof=1) + 1) - mu) / std


def stock_autocorr(stock, species=0, lag=1, mu=0, std=1):
    """The lag autocorrelation of a species' standardised observations (ddof = 1), divided by
    n_obs - 1 (lotka_volterra.py:243-256).  The device computes lags 1 and 2."""
    S = _device_summaries(stock)
    if S is not None:
        if lag not in (1, 2):
            raise ValueError('the device Lotka-Volterra summaries have the autocorrelations of lags '
                             '1 and 2, got lag {}'.format(lag))
        return _column(S, 2 + 2 * lag + species, mu, std)
    x = np.atleast_2d(stock[:, :, species])
    n = x.shape[1]
    z = (x - np.mean(x, axis=1, keepdims=True)) / np.std(x, axis=1, ddof=1, keepdims=True)
    return (np.sum(z[:, lag:] * z[:, :-lag], axis=1) / (n - 1) - mu) / std


def stock_crosscorr(stock, mu=0, std=1):
    """The cross-correlation of the two species' standardised observations; the standard deviations
    have ddof = 0 but the sum is divided by n_obs - 1, as in the reference
    (lotka_volterra.py:259-277)."""
    S = _device_summaries(stock)
    if S is not None:
        return _column(S, 8, mu, std)
    n = stock.shape[1]
    prey, pred = stock[:, :, 0], stock[:, :, 1]
    z_prey = (prey - np.mean(prey, axis=1, keepdims=True)) / np.std(prey, axis=1, keepdims=True)
    z_pred = (pred - np.mean(pred, axis=1, keepdims=True)) / np.std(pred, axis=1, keepdims=True)
    return (np.sum(z_prey * z_pred, axis=1) / (n - 1) - mu) / std


class ExpUniform:
    """log x ~ Uniform(a, b): pdf 1 / (x (b - a)) on [exp(a), exp(b)] (lotka_volterra.py:280-326).
    logpdf is the log of pdf, as for any ELFI distribution without its own logpdf."""

    @classmethod
    def rvs(cls, a, b, size=1, random_state=None):
        return np.exp(ss.uniform.rvs(loc=a, scale=b - a, size=size, random_state=random_state))

    @classmethod
    def pdf(cls, x, a, b):
        with np.errstate(divide='ignore'):
            p = np.where((x < np.exp(a)) | (x > np.exp(b)), 0, np.reciprocal(x))
            p /= (b - a)
        return p

    @classmethod
    def logpdf(cls, x, a, b):
        with np.errstate(divide='ignore', invalid='ignore'):
            return np.log(cls.pdf(x, a, b))


# ---------------------------------------------------------------------------- the task
def _true_params(true_params, observation_noise):
    if true_params is None:
        return [1.0, 0.005, 0.6, 50, 100, 10. if observation_noise else 0.]
    if observation_noise:
        if len(true_params) != 6:
            raise ValueError("Option observation_noise = True. Provide six input parameters.")
        return list(true_params)
    if len(true_params) != 5:
        raise ValueError("Option observation_noise = False. Provide five input parameters.")
    return list(true_params) + [0]


# the priors of lotka_volterra.py:193-202: (name, ExpUniform (a, b)) and (name, normal (loc, scale))
EXP_UNIFORM_PRIORS = (('r1', (-6., 2.)), ('r2', (-6., 2.)), ('r3', (-6., 2.)))
SIGMA_PRIOR = ('sigma', (np.log(0.5), np.log(50)))
NORMAL_PRIORS = (('prey0', (50, np.sqrt(50))), ('predator0', (100, np.sqrt(100))))


def _graph(m, exp_uniform, normal, simulator, y_obs, observation_noise):
    """Priors, simulator, summaries and distance of lotka_volterra.py:191-218."""
    priors = [em.Prior(exp_uniform, a, b, model=m, name=name) for name, (a, b) in EXP_UNIFORM_PRIORS]
    priors += [em.Prior(normal, loc, scale, model=m, name=name)
               for name, (loc, scale) in NORMAL_PRIORS]
    if observation_noise:
        name, (a, b) = SIGMA_PRIOR
        priors.append(em.Prior(exp_uniform, a, b, model=m, name=name))
    em.Simulator(simulator, *priors, observed=y_obs, name='LV')
    fns = [partial(stock_mean, species=0), partial(stock_mean, species=1),
           partial(stock_log_variance, species=0), partial(stock_log_variance, species=1),
           partial(stock_autocorr, species=0, lag=1), partial(stock_autocorr, species=1, lag=1),
           partial(stock_autocorr, species=0, lag=2), partial(stock_autocorr, species=1, lag=2),
           stock_crosscorr]
    sumstats = [em.Summary(fn, m['LV'], name=name) for fn, name in zip(fns, SUMMARY_NAMES)]
    em.Distance('euclidean', *sumstats, name='d')
    return m


def get_model(n_obs=50, true_params=None, observation_noise=False, seed_obs=None, **kwargs):
    """The Lotka-Volterra inference task of lotka_volterra.py:146-223: ExpUniform(-6, 2) priors on
    r1, r2, r3, normal priors on prey0 (50, sqrt 50) and predator0 (100, 10), with
    observation_noise an ExpUniform(log 0.5, log 50) prior on sigma; the simulator 'LV', the nine
    summaries and the Euclidean distance 'd'.  kwargs go to the simulator."""
    true_params = _true_params(true_params, observation_noise)
    kwargs['n_obs'] = n_obs
    y_obs = lotka_volterra(*true_params, random_state=np.random.RandomState(seed_obs), **kwargs)
    return _graph(em.new_model(), ExpUniform, 'normal', partial(lotka_volterra, **kwargs), y_obs,
                  observation_noise)


# ---------------------------------------------------------------------------- throughput mode
def lotka_volterra_device(r1, r2, r3, prey_init=50, predator_init=100, sigma=0., n_obs=16,
                          time_end=30., batch_size=1, random_state=None, return_full=False,
                          max_events=2 ** 20):
    """Device twin of lotka_volterra; returns a LazySimulation of shape (batch_size, n_obs, 2)
    whose summaries are the (batch_size, 9) tensor of ops.lv_summaries, computed once for all nine
    summary nodes.  materialize() gives the observations (float64 holding the int32 values; NaN
    for a row that needs more than max_events events or whose parameters the reference rejects)."""
    if return_full:
        raise ValueError('the device Lotka-Volterra simulator does not return the full event '
                         'history (its length per row is unbounded); use the host simulator')
    P = torch.stack(batch_columns((r1, r2, r3, prey_init, predator_init, sigma), batch_size), dim=1)
    key = batch_key(random_state)
    data = []

    def materialize():
        if not data:
            data.append(ops.sim_lotka_volterra(P, n_obs, time_end, seed=key,
                                               max_events=max_events)[0])
        return data[0]

    return LazySimulation((int(P.shape[0]), int(n_obs), 2),
                          lambda kind: ops.lv_summaries(materialize()), materialize)


class _DeviceExpUniform:
    """ExpUniform(a, b) drawn on the device as the reference builds it: exp of a uniform(a, b - a)
    draw (ops.prior_rvs); pdf / logpdf are ExpUniform's."""
    __name__ = 'device_ExpUniform'

    @staticmethod
    def rvs(a, b, size=1, random_state=None):
        n = int(np.prod(size))
        return torch.exp(ops.prior_rvs(prior_spec('uniform', [a, b - a]), n,
                                       batch_key(random_state)))

    pdf = ExpUniform.pdf
    logpdf = ExpUniform.logpdf


class DeviceProposal:
    """SMC proposals / prior density on the device for the Lotka-Volterra model (pass an instance as
    ``device_proposal=`` to SMC).  Columns in sorted parameter order.  ``rvs`` keeps the mixture
    draws inside the closed box where the prior density is positive: [exp(a), exp(b)] for the
    ExpUniform columns, the real line for the normal ones.  ``logpdf`` is the host ModelPrior's
    sum in that order: log(1 / x / (b - a)) inside the box and -inf outside for the ExpUniform
    columns, scipy's normal logpdf (ops.prior_logpdf) for the others."""

    def __init__(self, observation_noise=False):
        exp_priors = dict(EXP_UNIFORM_PRIORS + ((SIGMA_PRIOR,) if observation_noise else ()))
        normal_priors = dict(NORMAL_PRIORS)
        self.parameter_names = sorted(list(exp_priors) + list(normal_priors))
        self.columns = []       # (kind, parameters) per column
        lo, hi = [], []
        for name in self.parameter_names:
            if name in exp_priors:
                a, b = exp_priors[name]
                self.columns.append(('exp_uniform', (float(np.exp(a)), float(np.exp(b)),
                                                     float(b - a))))
                lo.append(float(np.exp(a)))
                hi.append(float(np.exp(b)))
            else:
                self.columns.append(('norm', np.asarray([prior_spec('norm', normal_priors[name])])))
                lo.append(-np.inf)
                hi.append(np.inf)
        self.box = (lo, hi)

    def rvs(self, means, cov, weights, size, key, cdf=None):
        return ops.gm_rvs(means, cov, weights, size, seed=key, support=2, box=self.box, cdf=cdf)

    def logpdf(self, params):
        x = ops._matrix(params)
        total = None
        for i, (kind, prm) in enumerate(self.columns):
            if kind == 'norm':
                term = ops.prior_logpdf(x[:, i:i + 1], prm)
            else:
                lo, hi, width = prm
                xi = x[:, i]
                outside = (xi < lo) | (xi > hi)
                term = torch.where(outside, torch.full_like(xi, -np.inf),
                                   torch.log(torch.reciprocal(xi) / width))
            total = term if total is None else total + term
        return total


def get_device_model(n_obs=50, true_params=None, observation_noise=False, seed_obs=None,
                     max_events=2 ** 20, **kwargs):
    """The Lotka-Volterra task in throughput mode: the graph of get_model with r1, r2, r3 (and
    sigma) drawn on the device as exp of a uniform, prey0 and predator0 from the device's normal
    prior, the device simulator (rows bounded by max_events events) and the nine summaries in one
    kernel; the Euclidean distance runs on the device.  The observed data comes from the host
    simulator.  Returns (model, DeviceProposal); pass the latter as ``device_proposal=`` to SMC."""
    if not ops.LV_SUMM_NOBS_MIN <= n_obs <= ops.LV_SUMM_NOBS_MAX:
        raise ValueError('the device Lotka-Volterra summaries take {} <= n_obs <= {}, got {}'.format(
            ops.LV_SUMM_NOBS_MIN, ops.LV_SUMM_NOBS_MAX, n_obs))
    true_params = _true_params(true_params, observation_noise)
    kwargs['n_obs'] = n_obs
    y_obs = lotka_volterra(*true_params, random_state=np.random.RandomState(seed_obs), **kwargs)
    simulator = partial(lotka_volterra_device, max_events=max_events, **kwargs)
    m = _graph(em.new_model(), _DeviceExpUniform, DevicePriorDistribution('norm'), simulator,
               y_obs, observation_noise)
    return m, DeviceProposal(observation_noise)
