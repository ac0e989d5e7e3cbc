"""Rounds of simulations at one parameter (elfi/methods/inference/parameter_inference.py:
ModelBased), the base of BSL and BOLFIRE.

A round runs n_sim_round simulations, batch_size at a time, at the parameter the method chose
for it.  The round's features go into one (n_sim_round, d) float64 device buffer (`_sim`), whatever
the model: lazy device simulations are materialised in place, host outputs uploaded once per batch.
When the round is full the method's `_process_simulated` runs, then `_init_round` prepares the
next round.  Runs on this rank only.

A method may run the rounds of `n_chains` chains side by side: each batch then holds batch_size
rows of every chain, chain c in rows [c batch_size, (c + 1) batch_size), at that chain's
parameter, and `_sim` is (n_chains, n_sim_round, d) (one chain keeps the (n_sim_round, d) view).
"""
import numpy as np
import torch

from . import device as dev
from . import model as em
from .samplers import ParameterInference


def feature_columns(batch, names, rows):
    """The outputs `names` of a batch as 2-d float64 device blocks of `rows` rows, in order (the
    columns of batch_to_arr2d): lazy simulations are materialised, host arrays uploaded."""
    blocks = []
    for name in names:
        v = batch[name]
        if hasattr(v, 'materialize'):
            v = v.materialize()
        t = v if dev.is_device_array(v) else dev.to_device(np.asarray(v, dtype=np.float64))
        if t.dtype != torch.float64:
            t = t.to(torch.float64)
        if t.dim() == 1:
            t = t[:, None]
        if t.dim() != 2 or t.shape[0] != rows:
            raise ValueError('Feature {} must be a ({}, k) array per batch, got shape {}'.format(
                name, rows, tuple(t.shape)))
        blocks.append(t)
    return blocks


def observed_row(model, feature_names):
    return np.column_stack([dev.to_host(model[node].observed) for node in feature_names])


def feature_list(feature_names):
    return [feature_names] if isinstance(feature_names, str) else list(feature_names)


class ModelBased(ParameterInference):
    """Base class of the methods that run each round of simulations at one parameter.
    Subclasses set D_MAX (the most features their device arithmetic takes) and provide
    `current_params`, `_process_simulated` and, when parameters change between rounds,
    `_init_round`."""

    D_MAX = None

    def __init__(self, model, n_sim_round, feature_names=None, batch_size=None, seed=None,
                 pool=None):
        model = model.model if isinstance(model, em.NodeReference) else model
        self.n_sim_round = int(n_sim_round)
        batch_size = batch_size or self.n_sim_round
        if self.n_sim_round % batch_size != 0:
            raise ValueError('n_sim_round must be a multiple of batch_size.')
        feature_names = feature_list(feature_names) if feature_names else [
            node for node in model.nodes
            if isinstance(model[node], em.Summary) and not node.startswith('_')]
        if not feature_names:
            raise ValueError('feature_names must include at least one item.')
        for node in feature_names:
            if node not in model.nodes:
                raise ValueError('Node {} not found in the model'.format(node))
        self.feature_names = feature_names
        self.n_chains = 1
        self._rows_per_chain = batch_size      # the context's batch size is n_chains times this
        super().__init__(model, model.parameter_names + feature_names, batch_size=batch_size,
                         seed=seed, pool=pool, distributed=False)
        self.observed = observed_row(self.model, feature_names)
        d = self.observed.size
        if not 1 <= d <= self.D_MAX:
            raise ValueError('{} takes 1 to {} features, got {}'.format(
                type(self).__name__, self.D_MAX, d))
        self._sim = None                  # (n_sim_round, d) or (n_chains, n_sim_round, d) features
        self.state['round'] = 0
        self.state['n_sim_round'] = 0

    def _init_state(self):
        self.state['n_batches'] = 0
        self.state['n_sim'] = 0
        self.state['round'] = 0
        self.state['n_sim_round'] = 0

    def set_objective(self, rounds):
        self.objective['round'] = rounds
        self.objective['n_batches'] = rounds * (self.n_sim_round // self._rows_per_chain)

    def infer(self, *args, **kwargs):
        if self.state['round'] > 0:
            self._init_round()
        return super().infer(*args, **kwargs)

    @property
    def current_params(self):
        raise NotImplementedError

    def prepare_new_batch(self, batch_index):
        params = np.repeat(np.atleast_2d(self.current_params), self._rows_per_chain, axis=0)
        return {p: params[:, i] for i, p in enumerate(self.parameter_names)}

    def update(self, batch, batch_index):
        super().update(batch, batch_index)
        self._merge_batch(batch)
        if self.state['n_sim_round'] == self.n_sim_round:
            self._process_simulated()
            self._end_round()

    def _end_round(self):
        self.state['round'] += 1
        if self.state['round'] < self.objective['round']:
            self._init_round()

    def _simulate_round(self):
        """Run the batches of the current round (as `iterate` does) and stop when its features
        are complete, without processing them: the caller evaluates the round and then calls
        `_end_round`.  A Testbench evaluates the rounds of several samplers in one call."""
        while self.state['n_sim_round'] < self.n_sim_round:
            batch_index = self._next_batch_index
            values = self.prepare_new_batch(batch_index)
            self._next_batch_index += 1
            batch = self._run_batch(batch_index, values)
            super().update(batch, batch_index)
            self._merge_batch(batch)

    def _init_round(self):
        self.state['n_sim_round'] = 0

    def _process_simulated(self):
        raise NotImplementedError

    def _merge_batch(self, batch):
        C, b, d = self.n_chains, self._rows_per_chain, self.observed.size
        if self._sim is None:
            sim = dev.empty((C, self.n_sim_round, d))
            self._sim = sim[0] if C == 1 else sim
        rounds = self._sim if self._sim.dim() == 3 else self._sim[None]
        row = self.state['n_sim_round']
        col = 0
        for block in feature_columns(batch, self.feature_names, self.batch_size):
            w = int(block.shape[1])
            if col + w > d:
                raise ValueError('The features are wider than their observed values ({})'.format(d))
            # chain c's rows of the batch go to its own round
            rounds[:, row:row + b, col:col + w] = block.reshape(C, b, w)
            col += w
        if col != d:
            raise ValueError('The features have {} columns, their observed values {}'.format(
                col, d))
        self.state['n_sim_round'] += b
