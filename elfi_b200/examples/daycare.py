"""Transmission of bacterial strains in day care centres (mirror of elfi/examples/daycare.py;
Numminen, Cheng, Gyllenberg & Corander 2013, and the BOLFI example of Gutmann & Corander 2016): an
SIS-type Markov jump process in each of n_dcc day care centres (DCCs) of n_ind children and
n_strains strains, simulated by Gillespie's direct method, and observed as the carriage of the first
n_obs children of each DCC.  Four summaries per DCC (Shannon index of the observed strains, number
of strains observed, prevalence of carriage and of multiple carriage) and a sorted-L1 distance.

The host path (daycare, the summaries, distance, get_model) consumes the batch's RandomState exactly
as the reference does, so it reproduces the reference's draws.  get_device_model is the same task in
throughput mode: the priors drawn on the device, the simulator on the device with the summaries
fused into it (one warp per row, one lane per DCC; Philox streams, statistical parity with the host
path at batch_size=1) and the distance on the device.

The summaries and the distance take host arrays (the reference's NumPy code), device tensors
(ops.daycare_summaries, ops.daycare_distance) and the lazy output of the device simulator; all
forms give the same values, except that the device's log in Shannon may make it differ from NumPy's
by an ulp or two (each log is within 1 ulp)."""
from functools import partial

import numpy as np
import torch

from .. import device as dev
from .. import model as em
from .. import ops
from ..priors import DeviceModelPrior
from ..throughput import LazySimulation, batch_columns, batch_key

SUMMARY_NAMES = ('Shannon', 'n_strains', 'prevalence', 'multi')


def daycare(t1, t2, t3, n_dcc=29, n_ind=53, n_strains=33, freq_strains_commun=None, n_obs=36,
            time_end=10., batch_size=1, random_state=None):
    """The day care simulator (daycare.py:16-141): (batch_size, n_dcc, n_obs, n_strains) bool
    carriage of the first n_obs children of each DCC.

    The whole batch steps together while any DCC of it is short of time_end.  A step draws
    exponential(1 / total hazard) (batch_size, n_dcc) for the waiting times, then uniform
    (batch_size, n_dcc, 1) for the transitions, which are picked in child-major order."""
    random_state = random_state or np.random

    t1 = np.asanyarray(t1).reshape((-1, 1, 1, 1))
    t2 = np.asanyarray(t2).reshape((-1, 1, 1, 1))
    t3 = np.asanyarray(t3).reshape((-1, 1, 1, 1))

    if freq_strains_commun is None:
        freq_strains_commun = np.full(n_strains, 0.1)

    prob_commun = t2 * freq_strains_commun
    state = np.zeros((batch_size, n_dcc, n_ind, n_strains), dtype=np.bool_)
    time = np.zeros((batch_size, n_dcc))
    n_factor = 1. / (n_ind - 1)
    gamma = 1.
    ind_b_dcc = [np.repeat(np.arange(batch_size), n_dcc), np.tile(np.arange(n_dcc), batch_size)]

    while np.any(time < time_end):
        with np.errstate(divide='ignore', invalid='ignore'):
            # E_s: the probability of sampling strain s
            prob_strain_adjust = np.nan_to_num(state / np.sum(state, axis=3, keepdims=True))
            prob_strain = np.sum(prob_strain_adjust, axis=2, keepdims=True)
        intrainfect_rate = t1 * (np.tile(prob_strain, (1, 1, n_ind, 1)) -
                                 prob_strain_adjust) * n_factor + 1e-9
        hazards = intrainfect_rate + prob_commun
        # co-infection is scaled by t3; carriers recover at rate gamma
        any_infection = np.any(state, axis=3, keepdims=True)
        hazards = np.where(any_infection, t3 * hazards, hazards)
        hazards[state] = gamma

        inv_sum_hazards = 1. / np.sum(hazards, axis=(2, 3), keepdims=True)
        probs = hazards * inv_sum_hazards
        delta_t = random_state.exponential(inv_sum_hazards[:, :, 0, 0])
        time = time + delta_t

        probs = probs.reshape((batch_size, n_dcc, -1))
        cumprobs = np.cumsum(probs[:, :, :-1], axis=2)
        x = random_state.uniform(size=(batch_size, n_dcc, 1))
        ind_transit = np.sum(x >= cumprobs, axis=2)
        ind_transit = ind_b_dcc + list(np.unravel_index(ind_transit.ravel(), (n_ind, n_strains)))
        state[tuple(ind_transit)] = np.logical_not(state[tuple(ind_transit)])

    return state[:, :, :n_obs, :]


# ---------------------------------------------------------------------------- summaries
def _device_summary(data, j):
    """Summary j (a (B, n_dcc) block of [Shannon | n_strains | prevalence | multi]) of lazy
    simulator output or device data; None for host data."""
    if isinstance(data, LazySimulation):
        S = data.summaries()
    elif dev.is_device_array(data):
        S = ops.daycare_summaries(data)
    else:
        return None
    n_dcc = S.shape[1] // ops.DC_NSUMM
    return S[:, j * n_dcc:(j + 1) * n_dcc]


def ss_shannon(data):
    """The Shannon index -sum p log p of the observed strains of each DCC (daycare.py:199-221)."""
    s = _device_summary(data, 0)
    if s is not None:
        return s
    total_obs = np.sum(data, axis=2, keepdims=True)
    with np.errstate(divide='ignore', invalid='ignore'):
        proportions = np.nan_to_num(total_obs / np.sum(total_obs, axis=3, keepdims=True))
    proportions[proportions == 0] = 1
    return (-np.sum(proportions * np.log(proportions), axis=3))[:, :, 0]


def ss_strains(data):
    """The number of strains observed in each DCC (daycare.py:224-239); float64 on the device."""
    s = _device_summary(data, 1)
    if s is not None:
        return s
    return np.sum(np.any(data, axis=2), axis=2)


def ss_prevalence(data):
    """The share of observed children carrying a strain (daycare.py:242-257)."""
    s = _device_summary(data, 2)
    if s is not None:
        return s
    return np.sum(np.any(data, axis=3), axis=2) / data.shape[2]


def ss_prevalence_multi(data):
    """The share of observed children carrying more than one strain (daycare.py:260-275)."""
    s = _device_summary(data, 3)
    if s is not None:
        return s
    return np.sum(np.sum(data, axis=3) > 1, axis=2) / data.shape[2]


def distance(*summaries, observed):
    """Mean L1 distance of the summaries, each divided by its observed maximum and sorted over the
    DCCs (daycare.py:278-312); device summaries give a device (B,) result (ops.daycare_distance)."""
    if any(dev.is_device_array(s) for s in summaries):
        n_dcc = int(summaries[0].shape[1])
        return ops.daycare_distance(em._stack_summaries(summaries), observed, n_dcc)
    summaries = np.stack(summaries)
    observed = np.stack(observed)
    n_ss, _, n_dcc = summaries.shape
    obs_max = np.max(observed, axis=2, keepdims=True)
    obs_max = np.where(obs_max == 0, 1, obs_max)
    y = np.sort(observed / obs_max, axis=2)
    x = np.sort(summaries / obs_max, axis=2)
    return np.sum(np.abs(x - y), axis=(0, 2)) / (n_ss * n_dcc)


# ---------------------------------------------------------------------------- the task
def _graph(m, simulator, y_obs):
    """Priors, simulator, summaries, distance and its log of daycare.py:173-191."""
    priors = [em.Prior('uniform', 0, 11, model=m, name='t1'),
              em.Prior('uniform', 0, 2, model=m, name='t2'),
              em.Prior('uniform', 0, 1, model=m, name='t3')]
    em.Simulator(simulator, *priors, observed=y_obs, name='DCC')
    sumstats = [em.Summary(fn, m['DCC'], name=name) for fn, name in zip(
        (ss_shannon, ss_strains, ss_prevalence, ss_prevalence_multi), SUMMARY_NAMES)]
    em.Discrepancy(distance, *sumstats, name='d')
    em.Operation(np.log, m['d'], name='logd')
    return m


def _observed(true_params, seed_obs, kwargs):
    if true_params is None:
        true_params = [3.6, 0.6, 0.1]
    return daycare(*true_params, random_state=np.random.RandomState(seed_obs), **kwargs)


def get_model(true_params=None, seed_obs=None, **kwargs):
    """The day care inference task of daycare.py:144-196: uniform priors t1 ~ U(0, 11),
    t2 ~ U(0, 2), t3 ~ U(0, 1), the simulator 'DCC', the four summaries, the distance 'd' and its
    log 'logd' (for BOLFI).  kwargs go to the simulator."""
    y_obs = _observed(true_params, seed_obs, kwargs)
    return _graph(em.new_model(), partial(daycare, **kwargs), y_obs)


# ---------------------------------------------------------------------------- throughput mode
def daycare_device(t1, t2, t3, n_dcc=29, n_ind=53, n_strains=33, freq_strains_commun=None,
                   n_obs=36, time_end=10., batch_size=1, random_state=None):
    """Device twin of daycare; returns a LazySimulation of shape (batch_size, n_dcc, n_obs,
    n_strains) whose summaries are the (batch_size, 4 n_dcc) tensor the simulator computes with
    them fused in, shared by the four summary nodes.  materialize() runs the simulator again from
    the same streams and gives the bool data.  Within a row every DCC takes as many transitions as
    the one that needs most to pass time_end, which is the reference's law at batch_size=1."""
    P = torch.stack(batch_columns((t1, t2, t3), batch_size), dim=1)
    key = batch_key(random_state)
    kw = dict(n_dcc=n_dcc, n_ind=n_ind, n_strains=n_strains,
              freq_strains_commun=freq_strains_commun, n_obs=n_obs, time_end=time_end, seed=key)
    return LazySimulation(
        (int(P.shape[0]), int(n_dcc), int(n_obs), int(n_strains)),
        lambda kind: ops.sim_daycare(P, **kw)[0],
        lambda: ops.sim_daycare(P, want_data=True, want_summaries=False, **kw)[1])


def get_device_model(true_params=None, seed_obs=None, **kwargs):
    """The day care task in throughput mode: the graph of get_model with the uniform priors drawn
    on the device, the device simulator with the four summaries fused into it, the distance on the
    device and 'logd' unchanged.  The observed data comes from the host simulator.  Returns
    (model, DeviceModelPrior); pass the latter as ``device_proposal=`` to SMC."""
    y_obs = _observed(true_params, seed_obs, kwargs)
    m = _graph(em.new_model(), partial(daycare_device, **kwargs), y_obs)
    dp = DeviceModelPrior(m)
    return dp.model, dp
