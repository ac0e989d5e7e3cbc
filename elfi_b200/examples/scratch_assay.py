"""Scratch assay model (mirror of elfi/examples/scratch_assay.py; Johnston et al. 2014, with the
summaries of Price et al. 2018): cells on an nrows x ncols lattice (27 x 36 by default) move and
proliferate in sequential, conflicting events; the lattice is observed every obs_interval and
summarised by the mismatch counts between consecutive observations and the final cell count.

pm (motility) and pp (proliferation) are inferred; the simulator 'sim' is the scalar cell_sim
vectorised with elfi_b200.tools.vectorize, its initial lattice a Constant parent, as in the
reference.

The host path (cell_sim, cell_summaries, get_model) consumes the batch's RandomState exactly as the
reference does, so it reproduces the reference's draws.  get_device_model is the same task in
throughput mode: the uniform priors drawn on the device (DeviceModelPrior), the lattice simulator
with the summaries fused on the device (one warp per row, Philox streams; the law of cell_sim).

cell_summaries takes host arrays (the reference's NumPy code), device tensors
(ops.scratch_assay_summaries) and the lazy output of the device simulator (the summaries computed
in the simulator); all forms give the same values, which are integers."""
import logging

import numpy as np
import torch

from .. import device as dev
from .. import model as em
from .. import ops
from .. import tools
from ..priors import DeviceModelPrior
from ..throughput import LazySimulation, batch_columns, batch_key

logger = logging.getLogger(__name__)

MOVES = ((1, 0), (-1, 0), (0, 1), (0, -1))     # row + 1, row - 1, col + 1, col - 1
DEFAULT_INIT = [27, 36, 100, 10]               # nrows, ncols, cells, rows they start in


def _random_init(nrows, ncols, ncell, nrows_init, random_state=None):
    """(nrows, ncols) lattice of ncell cells placed by one permutation of the first nrows_init
    rows."""
    random_state = random_state or np.random
    sites = np.zeros(nrows * ncols)
    sites[:ncell] = np.ones(ncell)
    head = nrows_init * ncols
    sites[:head] = random_state.permutation(sites[:head])
    return sites.reshape(nrows, ncols)


def _random_move(coords, nrows, ncols, random_state=None):
    """coords moved one site in a direction drawn with choice(4), clamped to the lattice."""
    random_state = random_state or np.random
    step = MOVES[random_state.choice(4)]
    target = np.array(coords) + step
    return np.minimum(np.maximum(target, 0), [nrows - 1, ncols - 1])


def cell_sim(pm, pp, init_arr=None, init_params=None, obs_period=12, obs_interval=1 / 12,
             tau=1 / 24, random_state=None):
    """One simulation: the lattice (nrows, ncols, num_obs + 1) at the start and after every
    obs_interval.  Each iteration snapshots the cells, then draws num_cells motility candidates
    (choice with replacement, then uniforms; kept when u < pm) and moves each kept one onto an
    empty neighbour, then the same for proliferation with pp, whose daughters fill the neighbour
    whether or not it is occupied.  A full lattice skips the iteration and its observation (the
    frames start as ones).  init_arr, or else a random lattice of init_params (default
    [27, 36, 100, 10])."""
    random_state = random_state or np.random
    if init_arr is None:
        lattice = _random_init(*(init_params or DEFAULT_INIT), random_state=random_state)
    else:
        lattice = np.copy(init_arr)
    nrows, ncols = lattice.shape
    num_iter = int(obs_period / tau)
    interval = int(obs_interval / tau)
    num_obs = int(num_iter / interval)
    frames = np.ones((num_obs + 1, nrows, ncols))
    frames[0] = np.copy(lattice)

    for it in range(num_iter):
        num_cells = int(np.sum(lattice))
        coords = np.transpose(np.array(np.where(lattice)))
        if num_cells == nrows * ncols:
            continue

        picked = random_state.choice(num_cells, size=num_cells)
        u = random_state.uniform(size=num_cells)
        for cell in picked[u < pm]:
            to = _random_move(coords[cell], nrows, ncols, random_state)
            if lattice[to[0], to[1]] == 0:
                lattice[coords[cell][0], coords[cell][1]] = 0
                lattice[to[0], to[1]] = 1
                coords[cell] = to

        picked = random_state.choice(num_cells, size=num_cells)
        u = random_state.uniform(size=num_cells)
        for cell in picked[u < pp]:
            to = _random_move(coords[cell], nrows, ncols, random_state)
            lattice[to[0], to[1]] = 1

        if (it + 1) % interval == 0:
            frames[int((it + 1) / interval)] = np.copy(lattice)

    return np.transpose(frames, (1, 2, 0))


def _device_summaries(x):
    """The summaries of lazy simulator output or device data; None for host data."""
    if isinstance(x, LazySimulation):
        return x.summaries()
    if dev.is_device_array(x):
        return ops.scratch_assay_summaries(x)
    return None


def cell_summaries(x):
    """(batch_size, num_obs + 1) of data (batch_size, nrows, ncols, num_obs + 1): the summed
    absolute differences between consecutive frames, then the cells of the last frame.  Boolean
    or unsigned host data is read as float64 (so that differences cannot wrap)."""
    s = _device_summaries(x)
    if s is not None:
        return s
    x = np.asarray(x)
    if x.dtype.kind in 'bu':
        x = x.astype(np.float64)
    ds = np.sum(np.abs((x[:, :, :, :-1] - x[:, :, :, 1:])), axis=(1, 2))
    count = np.sum(x[:, :, :, -1], axis=(1, 2))[:, None]
    return np.concatenate((ds, count), axis=1)


def _observed(true_params, init_arr, init_params, seed_obs):
    """(observed data (1, nrows, ncols, num_obs + 1), its first frame, the distance weights
    [1 / num_ds] * num_ds + [1], divided by the initial cell count squared)."""
    if true_params is None:
        true_params = [0.25, 0.002]
    obs = cell_sim(*true_params, init_arr, init_params,
                   random_state=np.random.RandomState(seed_obs))
    first = obs[:, :, 0]
    obs = obs[None, :]
    num_ds = cell_summaries(obs).size - 1
    num_init = np.sum(first)
    weis = np.concatenate((np.ones(num_ds) / num_ds, np.array([1]))) / num_init ** 2
    logger.info("Generated observations with true parameters pm: %g, pp: %g", *true_params)
    return obs, first, weis


def _graph(m, simulator, obs, init_arr, weis):
    """Priors, simulator, summary and distance of the reference's get_model."""
    em.Prior('uniform', 0, 1, model=m, name='pm')
    em.Prior('uniform', 0, 1, model=m, name='pp')
    em.Simulator(simulator, m['pm'], m['pp'], init_arr, name='sim', observed=obs)
    em.Summary(cell_summaries, m['sim'], name='sums')
    em.Distance('euclidean', m['sums'], w=weis, name='d')
    return m


def get_model(true_params=None, init_arr=None, init_params=None, seed_obs=None):
    """The scratch assay task: priors pm, pp ~ U(0, 1), the simulator 'sim' (cell_sim vectorised,
    the observed series' first frame as its initial lattice), the summary 'sums' and the weighted
    Euclidean distance 'd'.  true_params defaults to [0.25, 0.002]."""
    obs, first, weis = _observed(true_params, init_arr, init_params, seed_obs)
    return _graph(em.new_model(), tools.vectorize(cell_sim, constants=(2,)), obs, first, weis)


# ---------------------------------------------------------------------------- throughput mode
def scratch_assay_device(pm, pp, init_arr, obs_period=12, obs_interval=1 / 12, tau=1 / 24,
                         batch_size=1, random_state=None):
    """Device twin of the vectorised cell_sim: a LazySimulation of shape (batch_size, nrows,
    ncols, num_obs + 1) whose cell_summaries are computed in the simulator kernel; the frames are
    written (as bool) only by materialize()."""
    P = torch.stack(batch_columns((pm, pp), batch_size), dim=1)
    key = batch_key(random_state)
    init = ops._scratch_init(init_arr)
    nrows, ncols = (int(v) for v in init.shape)
    _, _, num_obs = ops.scratch_assay_steps(obs_period, obs_interval, tau)
    steps = dict(obs_period=obs_period, obs_interval=obs_interval, tau=tau, seed=key)
    return LazySimulation(
        (int(P.shape[0]), nrows, ncols, num_obs + 1),
        lambda kind: ops.sim_scratch_assay(P, init, **steps)[1],
        lambda: ops.sim_scratch_assay(P, init, want_data=True, want_summaries=False, **steps)[0])


def get_device_model(true_params=None, init_arr=None, init_params=None, seed_obs=None):
    """The scratch assay task in throughput mode: the graph of get_model with the uniform priors
    drawn on the device and the device simulator with the summaries fused into it.  The observed
    data, its summaries and the weights are computed on the host.  Returns (model,
    DeviceModelPrior); pass the latter as ``device_proposal=`` to SMC."""
    obs, first, weis = _observed(true_params, init_arr, init_params, seed_obs)
    nrows, ncols = first.shape
    if nrows * ncols > ops.SA_SITES_MAX:
        raise ValueError('the device scratch assay simulator takes a lattice of at most {} sites, '
                         'got {} x {}'.format(ops.SA_SITES_MAX, nrows, ncols))
    m = _graph(em.new_model(), scratch_assay_device, obs, first, weis)
    dp = DeviceModelPrior(m)
    return dp.model, dp
