"""Graph helpers (mirror of elfi/model/tools.py): ``vectorize`` turns a simulator written for one
parameter set into one that takes a batch, by calling it once per row, and
``external_operation`` turns a command line (a shell script or an executable) into an operation
that runs it on a subprocess.  ``cuda_simulator`` turns a CUDA function that simulates one row
into a throughput-mode simulator, and ``fused_summary`` reads the summaries it computes."""
import subprocess
from functools import partial

import numpy as np

from . import device as dev
from . import ops
from .model import get_sub_seed
from .throughput import LazySimulation, batch_columns, batch_key

__all__ = ['vectorize', 'external_operation', 'cuda_simulator', 'fused_summary']

USERSIM_SALT = 0x55534552   # "USER": the default salt of cuda_simulator's streams


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


def unpack_meta(*inputs, **kwinputs):
    """Update ``kwinputs`` with the keys and values of its ``meta`` dictionary; keyword inputs
    given explicitly win over meta keys of the same name."""
    if 'meta' in kwinputs:
        new_kwinputs = kwinputs['meta'].copy()
        new_kwinputs.update(kwinputs)
        kwinputs = new_kwinputs
    return inputs, kwinputs


def prepare_seed(*inputs, **kwinputs):
    """Set ``kwinputs['seed']`` from its ``random_state`` (a NumPy RandomState): sub seed
    ``index_in_batch`` (0 when absent) of the first word of the state, so that every row of a
    batch gets its own seed."""
    if 'random_state' in kwinputs:
        seed = kwinputs['random_state'].get_state()[1][0]
        kwinputs['seed'] = get_sub_seed(seed, kwinputs.get('index_in_batch') or 0)
    return inputs, kwinputs


def stdout_to_array(stdout, *inputs, sep=' ', dtype=None, **kwinputs):
    """One row of stdout as a NumPy array (``np.fromstring`` with ``sep``)."""
    return np.fromstring(stdout, dtype=dtype, sep=sep)


def run_external(command, *inputs, process_result=None, prepare_inputs=None, stdout=True,
                 subprocess_kwargs=None, **kwinputs):
    """Run ``command`` on a subprocess and return ``process_result`` of what it gave.

    The meta keys are merged into the keyword inputs (:func:`unpack_meta`), a ``seed`` is derived
    from ``random_state`` (:func:`prepare_seed`), ``prepare_inputs`` may rewrite the inputs, and
    the command is ``command.format(*inputs, **kwinputs)``.  It runs with
    ``subprocess.run(shell=True, check=True)`` updated by ``subprocess_kwargs``, so a failing
    command raises CalledProcessError.  See :func:`external_operation`."""
    inputs, kwinputs = unpack_meta(*inputs, **kwinputs)
    inputs, kwinputs = prepare_seed(*inputs, **kwinputs)
    if prepare_inputs:
        inputs, kwinputs = prepare_inputs(*inputs, **kwinputs)
    try:
        command = command.format(*inputs, **kwinputs)
    except KeyError as e:
        raise KeyError('The requested keyword {} was not passed to the external '
                       'operation: "{}".'.format(str(e), command))
    kwargs = dict(shell=True, check=True)
    kwargs.update(subprocess_kwargs or {})
    completed_process = subprocess.run(command, **kwargs)
    if stdout:
        completed_process = completed_process.stdout
    return process_result(completed_process, *inputs, **kwinputs)


def external_operation(command, process_result=None, prepare_inputs=None, sep=' ', stdout=True,
                       subprocess_kwargs=None):
    """Wrap an external command (a shell script, an executable) as an operation, e.g. a simulator.

    Parameters
    ----------
    command : str
        The command line, with Python format fields for the inputs, e.g.
        ``"myscript.sh {0} {batch_size} --seed {seed}"``.  An operation that receives
        ``random_state`` also gets a ``seed`` keyword (:func:`prepare_seed`), and an operation
        with ``uses_meta`` the meta keys (``model_name``, ``batch_index``, ``submission_index``,
        ...).
    process_result : callable, np.dtype or str, optional
        ``output = process_result(result, *inputs, **kwinputs)``, where result is the stdout, or
        the ``subprocess.CompletedProcess`` when ``stdout`` is False.  The default converts
        stdout with ``np.fromstring(stdout, sep=sep)``; a dtype or its name casts it to that type.
    prepare_inputs : callable, optional
        ``inputs, kwinputs = prepare_inputs(*inputs, **kwinputs)``, called before the command is
        formatted (to write an input file, say).
    sep : str, optional
        The separator of the default ``process_result``.
    stdout : bool, optional
        Pass ``process_result`` the stdout (True, forced for the default handler) or the
        ``CompletedProcess``.
    subprocess_kwargs : dict, optional
        Options of ``subprocess.run``, over the defaults ``shell=True, check=True``.

    Example::

        op = elfi_b200.tools.external_operation('echo 1 {0}', process_result='int8')
        sim = elfi_b200.Simulator(op, elfi_b200.Constant(123))
        sim.generate()      # array([  1, 123], dtype=int8)
    """
    if process_result is None or isinstance(process_result, (str, np.dtype)):
        fromstring_kwargs = dict(sep=sep)
        if isinstance(process_result, (str, np.dtype)):
            fromstring_kwargs['dtype'] = str(process_result)
        process_result = partial(stdout_to_array, **fromstring_kwargs)
        stdout = True
    if stdout is True:
        subprocess_kwargs = dict(subprocess_kwargs or {})
        subprocess_kwargs['stdout'] = subprocess.PIPE
    return partial(run_external, command, process_result=process_result,
                   prepare_inputs=prepare_inputs, stdout=stdout,
                   subprocess_kwargs=subprocess_kwargs)


def cuda_simulator(source, n_params, n_out, n_summaries=0, salt=USERSIM_SALT):
    """A throughput-mode simulator from CUDA source that simulates one row.

    ``source`` defines ``__device__ void simulate(const double* theta, elfi::RowStream& rng,
    double* y)``, which writes the ``n_out`` values ``y[0 .. n_out)`` of one row from its
    ``n_params`` parameters, and, when ``n_summaries`` > 0, ``__device__ void summarise(const
    double* y, double* s)``, which writes that row's summaries.  ``rng`` is the row's Philox
    stream: ``rng.normal2(m, n0, n1)`` / ``rng.uniform2(m, u0, u1)`` give the two normals /
    uniforms of block m, ``rng.block(m)`` its raw words, and ``rng.next_normal()`` /
    ``rng.next_uniform()`` draw blocks in order.  ``elfi::n_params``, ``elfi::n_out`` and
    ``elfi::n_sum`` are the shapes.  elfi_b200/csrc/usersim_rt.cuh states the contract.

    The source is compiled for the H100 (NVRTC, sm_90a) on the first call on a device, and the
    compiled code is kept for the same source, shapes and salt.  A compile error raises
    ElfiB200Error carrying NVRTC's log.

    Returns ``simulator(*params, batch_size=1, random_state=None)``, whose output is a
    LazySimulation of shape (batch_size, n_out): ``summaries()`` runs simulate and summarise in
    one kernel without writing the data (when n_out <= ops.USERSIM_LOCAL_MAX), and
    ``materialize()`` writes the data.  Each call draws its Philox key from ``random_state``, as
    the built-in throughput-mode simulators do, so a run is a function of its seed.
    ``simulator.summarise(y)`` gives the summaries of data such as the observed rows.

    Example::

        sim = elfi_b200.tools.cuda_simulator(MA2_SOURCE, 2, 100, n_summaries=2)
        elfi_b200.Simulator(sim, m['t1'], m['t2'], observed=y_obs, name='MA2')
        elfi_b200.Summary(elfi_b200.tools.fused_summary(0, sim), m['MA2'], name='S1')
    """
    if not isinstance(source, str) or not source.strip():
        raise ValueError('the simulator source must be a non-empty string')
    n_params, n_out, n_summaries, salt = ops.usersim_shapes(n_params, n_out, n_summaries, salt)
    compiled = {}

    def on_device():
        device = dev.current_device()
        if device not in compiled:
            compiled[device] = ops.usersim_compile(source, n_params, n_out, n_summaries, salt)
        return compiled[device]

    def summaries(sim, cols, key, kind):
        if n_summaries == 0:
            raise ValueError('this CUDA simulator has no summaries (n_summaries = 0)')
        return ops.usersim_run(sim, cols, seed=key)[1]

    def simulator(*params, batch_size=1, random_state=None):
        if len(params) != n_params:
            raise ValueError('this CUDA simulator takes {} parameters, got {}'.format(
                n_params, len(params)))
        cols = batch_columns(params, batch_size)
        key = batch_key(random_state)
        sim = on_device()
        return LazySimulation(
            (int(cols[0].numel()), n_out), partial(summaries, sim, cols, key),
            lambda: ops.usersim_run(sim, cols, seed=key, want_data=True, want_summaries=False)[0])

    simulator.summarise = lambda y: ops.usersim_summarise(on_device(), y)
    return simulator


def fused_summary(columns, simulator=None):
    """A summary operation that reads columns of the summaries a :func:`cuda_simulator` computes.

    ``columns`` is one column index (the summary is (batch,)) or a list of them ((batch, k)).  The
    summaries of a simulator output come from its kernel.  Data that did not come from the
    simulator, such as the observed data, is summarised by ``simulator.summarise``, so pass the
    simulator when the model has observed data; without it such data raises ValueError."""
    index = int(columns) if np.ndim(columns) == 0 else [int(c) for c in columns]

    def summary(x):
        if isinstance(x, LazySimulation):
            S = x.summaries()
        elif simulator is not None:
            S = simulator.summarise(x)
        else:
            raise ValueError('fused_summary reads the summaries of a cuda_simulator output; '
                             'to summarise other data, such as the observed data, give it the '
                             'simulator: fused_summary(columns, simulator)')
        return S[:, index]
    return summary
