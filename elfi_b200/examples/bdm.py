"""The birth-death-mutation (BDM) model of tuberculosis transmission (mirror of
elfi/examples/bdm.py; Tanaka et al. 2006), the model of Lintusaari et al. 2016 with summary T1.

A population of one grows by births (rate alpha), shrinks by deaths (rate delta) and founds new
genotype clusters by mutation (rate tau) until it exceeds N or dies out; the data are the N
cluster sizes.  Summaries T1 (clusters per individual) and T2 (the gene diversity with n = 20).

The host path (get_model) runs the reference's C++ simulator as an outside executable `bdm` in the
working directory, through tools.external_operation, with an input and an output file per batch,
so it reproduces the reference's draws.  The reference ships that executable's source with its
examples (elfi/examples/cpp/bdm.cpp; `make` there builds it); this package does not.
get_device_model is the same task in throughput mode: the prior drawn on the device, the simulator
on the device (one lane per row, lanes refilled with new rows as theirs finish; Philox streams)
with T1 and T2 fused into it, and the distance on the device.  It needs no executable.

The two modes agree in law at parameters with four decimals: the host path writes its parameters
to the input file as %.4f, as the reference does, while the device takes them as given.

References
----------
- Jarno Lintusaari, Michael U. Gutmann, Ritabrata Dutta, Samuel Kaski, Jukka Corander;
  Fundamentals and Recent Developments in Approximate Bayesian Computation.
  Syst Biol 2017; 66 (1): e66-e82. doi: 10.1093/sysbio/syw077
- Mark M. Tanaka et al.; Using approximate Bayesian computation to estimate tuberculosis
  transmission parameters from genotype data. Genetics 2006; 173 (3): 1511-1520.
"""
import os
import warnings
from functools import partial

import numpy as np
import torch

from .. import device as dev
from .. import model as em
from .. import ops
from .. import tools
from ..priors import DeviceModelPrior
from ..throughput import LazySimulation, batch_columns, batch_key

MAX_EVENTS = 2 ** 24    # events per device row; the example's prior needs a few thousand at most
# the observed cluster sizes of Lintusaari et al. 2016 (N = 20)
LINTUSAARI_DATA = (6, 3, 2, 2, 1, 1, 1, 1, 1, 1, 1)


def prepare_inputs(*inputs, **kwinputs):
    """Write the input file of the bdm executable, one row "alpha delta tau N" per simulation
    (%.4f for the rates), named after the batch's meta, and add ``filename`` and
    ``output_filename`` to kwinputs.  The signature is that of tools.external_operation."""
    alpha, delta, tau, N = inputs
    meta = kwinputs['meta']
    param_array = np.vstack(
        [(a, d, t, n) for (a, d, t, n) in np.broadcast(alpha, delta, tau, N)])
    # a unique file name per batch, for parallel runs
    filename = '{model_name}_{batch_index}_{submission_index}.txt'.format(**meta)
    np.savetxt(filename, param_array, fmt='%.4f %.4f %.4f %d')
    kwinputs['filename'] = filename
    kwinputs['output_filename'] = filename[:-4] + '_out.txt'
    return inputs, kwinputs


def process_result(completed_process, *inputs, **kwinputs):
    """Read the simulations (int16 cluster sizes) from the output file and remove both files.
    The signature is that of tools.external_operation."""
    output_filename = kwinputs['output_filename']
    simulations = np.loadtxt(output_filename, dtype='int16')
    os.remove(kwinputs['filename'])
    os.remove(output_filename)
    return simulations


# the outside executable as an operation
BDM = tools.external_operation('./bdm {filename} --seed {seed} --mode 1 > {output_filename}',
                               prepare_inputs=prepare_inputs, process_result=process_result,
                               stdout=False)


def _device_summaries(clusters, n=None):
    """The (B, 2) [T1, T2] of lazy simulator output or device data; None for host data.  n=None
    takes the lazy output's fused summaries, whatever T2 argument they were computed with."""
    if isinstance(clusters, LazySimulation):
        return clusters.summaries(n)
    if dev.is_device_array(clusters):
        return ops.bdm_summaries(clusters, 20 if n is None else n)
    return None


def T1(clusters):
    """The number of clusters over the population size."""
    S = _device_summaries(clusters)
    if S is not None:
        return S[:, 0]
    clusters = np.atleast_2d(clusters)
    return np.sum(clusters > 0, axis=1) / np.sum(clusters, axis=1)


def T2(clusters, n=20):
    """1 - sum((cluster size / n)^2): the gene diversity for a sample of n."""
    S = _device_summaries(clusters, n)
    if S is not None:
        return S[:, 1]
    clusters = np.atleast_2d(clusters)
    return 1 - np.sum((clusters / n)**2, axis=1)


def _observed_lintusaari(N):
    y = np.zeros(N, dtype='int16')
    y[:len(LINTUSAARI_DATA)] = LINTUSAARI_DATA
    return y


def _graph(m, simulator, delta, tau, N, y):
    """Prior, simulator, T1 and the L1 distance of bdm.py:121-125."""
    em.Prior('uniform', .005, 2, model=m, name='alpha')
    em.Simulator(simulator, m['alpha'], delta, tau, N, observed=y, name='BDM')
    em.Summary(T1, m['BDM'], name='T1')
    em.Distance('minkowski', m['T1'], p=1, name='d')
    return m


def get_model(alpha=0.2, delta=0, tau=0.198, N=20, seed_obs=None):
    """The model of Lintusaari et al. 2016 (bdm.py:88-138): alpha ~ U(0.005, 2.005), the
    simulator 'BDM' (the executable `bdm`, expected in the working directory), T1 and the L1
    distance 'd'.  seed_obs=None with N = 20 observes the data of Lintusaari et al.; otherwise
    the observation is simulated at (alpha, delta, tau, N) with RandomState(seed_obs), with the
    meta of batch 0 of a model named 'bdm' (the reference calls BDM without meta there and
    raises KeyError)."""
    if seed_obs is None and N == 20:
        y = _observed_lintusaari(N)
    else:
        y = BDM(alpha, delta, tau, N, random_state=np.random.RandomState(seed_obs),
                meta=dict(model_name='bdm', batch_index=0, submission_index=0))
    m = _graph(em.new_model('bdm'), BDM, delta, tau, N, y)
    m['BDM'].uses_meta = True
    if not os.path.isfile('bdm') and not os.path.isfile('bdm.exe'):
        warnings.warn("This model uses an external simulator `bdm` implemented in C++ that needs "
                      "to be compiled and copied to your working directory. We could not find it "
                      "in your current working directory. Its source is elfi/examples/cpp/bdm.cpp "
                      "of the reference package ELFI.", RuntimeWarning)
    return m


# ---------------------------------------------------------------------------- throughput mode
def bdm_device(alpha, delta, tau, N, n_t2=20, batch_size=1, random_state=None,
               max_events=MAX_EVENTS):
    """Device twin of BDM; returns a LazySimulation of shape (batch_size, N) whose summaries are
    the (batch_size, 2) [T1, T2 (n = n_t2)] tensor the simulator computes with them fused in.
    materialize() runs the simulator again from the same streams and gives the int16 cluster
    sizes.  A row with invalid rates, or still running after max_events events, has counts of -1
    and NaN summaries (ops.sim_bdm)."""
    N = int(np.asarray(N).reshape(-1)[0])
    P = torch.stack(batch_columns((alpha, delta, tau), batch_size), dim=1)
    key = batch_key(random_state)
    kw = dict(seed=key, max_events=max_events)
    data, fused = [], []

    def materialize():
        if not data:
            data.append(ops.sim_bdm(P, N, want_summaries=False, **kw)[0])
        return data[0]

    def summarise(n):
        if n is None or n == n_t2:
            if not fused:
                fused.append(ops.sim_bdm(P, N, n=n_t2, want_data=False, **kw)[1])
            return fused[0]
        return ops.bdm_summaries(materialize(), n)

    return LazySimulation((int(P.shape[0]), N), summarise, materialize)


def get_device_model(alpha=0.2, delta=0, tau=0.198, N=20, seed_obs=None, max_events=MAX_EVENTS):
    """The BDM task in throughput mode: the graph of get_model with the uniform prior drawn on the
    device, the device simulator with T1 and T2 fused into it (rows bounded by max_events events)
    and the L1 distance on the device.  seed_obs=None with N = 20 observes the data of Lintusaari
    et al.; otherwise the device simulator draws the observation with the key of
    RandomState(seed_obs), so no executable is needed.  Returns (model, DeviceModelPrior); pass the
    latter as ``device_proposal=`` to SMC."""
    if seed_obs is None and N == 20:
        y = _observed_lintusaari(N)
    else:
        lazy = bdm_device(alpha, delta, tau, N, random_state=np.random.RandomState(seed_obs),
                          max_events=max_events)
        y = lazy.materialize().cpu().numpy()[0]
    simulator = partial(bdm_device, max_events=max_events)
    m = _graph(em.new_model('bdm'), simulator, delta, tau, N, y)
    dp = DeviceModelPrior(m)
    return dp.model, dp
