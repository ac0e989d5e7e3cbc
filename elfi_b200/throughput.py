"""Host plumbing shared by the throughput-mode examples: the Philox key of a node, the parameter
columns of a batch, and the lazy simulator output whose summaries come from the simulator kernel."""
import numpy as np

from . import device as dev


def batch_key(random_state):
    """The Philox key of one node of a batch: one draw from the batch's RandomState (np.random
    when none is given)."""
    random_state = random_state or np.random
    return int(random_state.randint(2 ** 31 - 1))


def batch_columns(values, batch_size):
    """One (n,) float64 device vector per simulator argument: device tensors are flattened in place
    (no copy; the ops wrappers make their inputs contiguous), scalars and host arrays are flattened,
    broadcast to batch_size and uploaded."""
    return [v.reshape(-1) if dev.is_device_array(v) else
            dev.to_device(np.broadcast_to(np.asarray(v, dtype=np.float64).reshape(-1),
                                          (batch_size,)).copy())
            for v in values]


class LazySimulation:
    """Simulator output whose summaries are computed in the simulator kernel, so the data is only
    written when ``materialize()`` is called.  ``summarise(kind)`` runs once per kind: the summary
    nodes of one simulator get columns of the same tensor, which the distance reads in place.

    ``euclidean``, when given, is the Euclidean distance of the data to an observed row computed in
    the simulator kernel: ``euclidean(obs, thresholds) -> (d, idx)`` with the contract of
    ``ops.dist_euclid(materialize(), obs, thresholds=thresholds)``.  A Euclidean ``Distance`` whose
    single parent is this output uses it; any other consumer of the data materialises it."""

    def __init__(self, shape, summarise, materialize, euclidean=None):
        self.shape = tuple(shape)
        self.ndim = len(self.shape)
        self._summarise = summarise
        self.materialize = materialize
        self.euclidean = euclidean
        self._summaries = {}

    def __len__(self):
        return self.shape[0]

    def summaries(self, kind=None):
        if kind not in self._summaries:
            self._summaries[kind] = self._summarise(kind)
        return self._summaries[kind]
