"""Graph helpers (mirror of elfi/model/tools.py): ``vectorize`` turns a simulator written for one
parameter set into one that takes a batch, by calling it once per row.

``external_operation`` (running an outside executable per row) is not provided."""
from functools import partial

import numpy as np

__all__ = ['vectorize']


def _is_array(x):
    """A batch input: anything with a shape and at least one dimension (lists, tuples and 0-d
    arrays are passed whole)."""
    return hasattr(x, 'shape') and x.ndim > 0


def run_vectorized(operation, *inputs, constants=None, dtype=None, batch_size=None, **kwargs):
    """Call ``operation`` once per row of the batch and collect the outputs.

    Inputs whose positional index is in ``constants``, and inputs that are not arrays, are passed
    whole to every call; every other input is indexed by the row.  Their lengths must agree (and
    agree with ``batch_size`` when given), else ValueError.  Without array inputs or batch_size
    the batch has one row.  Every call receives the same keyword arguments (so one random_state is
    consumed row after row); a ``meta`` dictionary among them gets ``index_in_batch`` set to the
    row before each call.

    Returns ``np.array(outputs, dtype=dtype)``, or with ``dtype=False`` a 1-d object array holding
    the outputs as returned."""
    constants = set() if constants is None else set(constants)
    batched = []
    for i, value in enumerate(inputs):
        if i in constants:
            continue
        if not _is_array(value):
            constants.add(i)
            continue
        if batch_size is None:
            batch_size = len(value)
        elif len(value) != batch_size:
            raise ValueError('Batch size {} does not match the length {} of input {}. Mark the '
                             'inputs that are passed whole with the `constants` argument of '
                             'vectorize.'.format(batch_size, len(value), i))
        batched.append(i)
    if batch_size is None:
        batch_size = 1

    outputs = np.empty(batch_size, dtype=object) if dtype is False else [None] * batch_size
    for row in range(batch_size):
        args = [value[row] if i in batched else value for i, value in enumerate(inputs)]
        if 'meta' in kwargs:
            kwargs['meta']['index_in_batch'] = row
        outputs[row] = operation(*args, **kwargs)
    if dtype is False:
        return outputs
    return np.array(outputs, dtype=dtype)


def vectorize(operation, constants=None, dtype=None):
    """A batch version of ``operation``, which takes one parameter set per call.

    Parameters
    ----------
    operation : callable
    constants : tuple or list of int, optional
        Positional indices of the inputs passed whole to every call, e.g. ``(2,)`` for a
        simulator whose third argument is an initial state.  Inputs that are not arrays are
        passed whole anyway.
    dtype : np.dtype or False, optional
        None lets ``np.array`` convert the list of outputs; False keeps the outputs as returned,
        in a 1-d object array.

    The rows run one after another in Python, so this suits simulators that cannot be written
    for a batch; a batched simulator is much faster.

    Example::

        sim = elfi_b200.tools.vectorize(cell_sim, constants=(2,))
        elfi_b200.Simulator(sim, m['pm'], m['pp'], init_arr, name='sim', observed=obs)
    """
    return partial(run_vectorized, operation, constants=constants, dtype=dtype)
