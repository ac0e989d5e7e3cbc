"""Host side of the operator (node) API for the hot path.

The public names, argument meanings and error types are those of elfi/model/elfi_model.py (the
drop-in boundary asks for that); the machinery behind them is this package's own:

* a model is a table ``name -> NodeRecord`` (operation or constant, a flag word, the ordered
  parent names, a free attribute dict) -- no graph library;
* ``compile_plan`` lowers the table once per inference into a :class:`Plan`: a flat list of
  :class:`Step` s in the reference's execution order, with the observed twins and the
  ``_batch_size`` / ``_meta`` / ``_random_state`` inputs already wired in;
* ``Plan.run`` executes one batch: it binds the per-batch inputs, skips every step whose value is
  already known (constants, observed data, pool hits, cached observed twins) and calls the rest.
  Summary / Distance steps launch CUDA kernels and hand device arrays to each other.

Behaviour that must equal the reference's because results depend on it bit for bit:
  the execution order of the compiled graph  elfi/executor.py:162-246 (golden: topo_orders.json)
  the per-batch sub-seeded RandomState       elfi/loader.py:131-178, elfi/utils.py:71-127
  observed twins / feeder inputs / pruning   elfi/compiler.py:32-235
  node semantics                             elfi/model/elfi_model.py:477-1151
Not provided: pickling, naming a node after the caller's assignment target, other clients.
"""
import uuid
from functools import partial

import numpy as np
import scipy.stats as ss

from . import device as dev
from . import ops
from .throughput import LazySimulation

# ---- node flags -----------------------------------------------------------------------------
STOCHASTIC = 1        # consumes the batch RandomState
OBSERVABLE = 2        # has an observed twin computed from the observed data
TAKES_OBSERVED = 4    # receives the tuple of its parents' observed twins as `observed=`
TAKES_BATCH_SIZE = 8
TAKES_META = 16
TAKES_ACCEPT = 32     # a device distance that can fuse the acceptance test (`accept=`)
PARAMETER = 64

BATCH_SIZE_INPUT, META_INPUT, RANDOM_STATE_INPUT = '_batch_size', '_meta', '_random_state'
_MISSING = object()

_SCIPY_SHORTHAND = {'normal': 'norm', 'exponential': 'expon', 'unif': 'uniform', 'bin': 'binom',
                    'binomial': 'binom'}


def scipy_from_str(name):
    key = name.lower()
    return getattr(ss, _SCIPY_SHORTHAND.get(key, key))


def random_name(length=4, prefix=''):
    return prefix + uuid.uuid4().hex[:length]


def observed_name(name):
    return '_' + name + '_observed'


def is_observed_name(name):
    return isinstance(name, str) and len(name) > 10 and name[0] == '_' and \
        name.endswith('_observed')


def is_array(output):
    return getattr(output, 'ndim', 0) > 0 and hasattr(output, 'shape')


def get_sub_seed(seed, sub_seed_index, high=2 ** 31, cache=None):
    """Sub seed number `sub_seed_index` of `seed`; bit-identical to elfi/utils.py:71-127
    (goldens in tests/golden/meta.json).

    The sub seeds of a seed are the distinct values of the uint32 stream
    ``RandomState(seed).randint(high)`` in order of first appearance; the stream is read in
    chunks of "as many as are still missing", which fixes how far it has advanced."""
    if isinstance(seed, np.random.RandomState):
        raise ValueError('Seed cannot be a random state')
    if sub_seed_index >= high:
        raise ValueError('Sub seed index {} is out of range'.format(sub_seed_index))
    wanted = sub_seed_index + 1
    stream, distinct = None, None
    if cache and len(cache['seen']) < wanted:
        stream, distinct = cache['random_state'], cache['seen']
    if stream is None:
        stream, distinct = np.random.RandomState(seed), set()
    chunk = None
    while len(distinct) < wanted:
        chunk = stream.randint(high, size=wanted - len(distinct), dtype='uint32')
        distinct.update(chunk)
    if cache is not None:
        cache['random_state'], cache['seen'] = stream, distinct
    return chunk[-1]


class ComputationContext:
    """What all batches of one inference share: batch size, master seed, an optional output
    pool, per-inference caches.  A pool that already carries a context supplies (and pins)
    batch size and seed (elfi/model/elfi_model.py:126-208)."""

    def __init__(self, batch_size=None, seed=None, pool=None):
        pinned = pool is not None and pool.has_context
        if pinned:
            batch_size = self._agree('batch_size', batch_size, pool.batch_size)
            seed = self._agree('seed', seed, pool.seed)
        if seed is None:
            seed = np.random.RandomState().get_state()[1][1]
        self.batch_size = batch_size or 1
        self.seed = seed
        self.pool = pool
        self.num_submissions = 0
        self.caches = {'plan': {}, 'sub_seed': {}}
        if pool is not None and not pinned:
            pool.set_context(self)

    @staticmethod
    def _agree(what, given, pooled):
        if given is not None and given != pooled:
            raise ValueError('Pool {0} differs from the given {0}!'.format(what))
        return pooled

    def callback(self, batch, batch_index):
        """A finished batch goes to the pool."""
        if self.pool is not None:
            self.pool.add_batch(batch, batch_index)


# ------------------------------------------------------------------------------------- model
class NodeRecord:
    """One row of the model table."""
    __slots__ = ('cls', 'op', 'constant', 'flags', 'inputs', 'attrs')

    def __init__(self, cls, op=None, constant=_MISSING, flags=0, attrs=None):
        self.cls = cls
        self.op = op
        self.constant = constant
        self.flags = flags
        self.inputs = []            # parent names, positional order
        self.attrs = {} if attrs is None else attrs

    def has(self, flag):
        return bool(self.flags & flag)

    def set(self, flag, on=True):
        self.flags = (self.flags | flag) if on else (self.flags & ~flag)

    def twin(self):
        """Same node, own parent list (model copies share operations and attribute dicts)."""
        rec = NodeRecord(self.cls, self.op, self.constant, self.flags, self.attrs)
        rec.inputs = list(self.inputs)
        return rec


_default_model = None


def get_default_model():
    global _default_model
    if _default_model is None:
        _default_model = ElfiModel()
    return _default_model


def set_default_model(model=None):
    global _default_model
    if model is not None and not isinstance(model, ElfiModel):
        raise ValueError('{} is not an instance of ElfiModel'.format(model))
    _default_model = ElfiModel() if model is None else model


def new_model(name=None, set_default=True):
    model = ElfiModel(name=name)
    if set_default:
        set_default_model(model)
    return model


class ElfiModel:
    """The node table of one generative model plus its observed data."""

    def __init__(self, name=None, observed=None):
        self.name = name or 'model_' + random_name()
        self._records = {}
        self._observed = {}
        if observed:
            self.observed = observed

    @property
    def observed(self):
        return self._observed

    @observed.setter
    def observed(self, observed):
        if not isinstance(observed, dict):
            raise ValueError('Observed data must be a dictionary {node name: data}')
        self._observed = observed

    # -- table access ---------------------------------------------------------------------
    @property
    def nodes(self):
        return list(self._records)

    def has_node(self, name):
        return name in self._records

    def record(self, name):
        return self._records[name]

    def get_parents(self, name):
        return list(self._records[name].inputs)

    def get_children(self, name):
        return [n for n, rec in self._records.items() if name in rec.inputs]

    def insert(self, name, record, parents=()):
        if name in self._records:
            raise ValueError('Node {} already exists'.format(name))
        for p in parents:
            if p not in self._records:
                raise ValueError('Parent {} does not exist'.format(p))
        record.inputs = list(parents)
        self._records[name] = record

    def remove_node(self, name):
        """Drop a node, its observed data and the hidden constants only it was using."""
        rec = self._records.pop(name)
        self._observed.pop(name, None)
        for other in self._records.values():
            if name in other.inputs:
                other.inputs = [p for p in other.inputs if p != name]
        for p in rec.inputs:
            if p.startswith('_') and p in self._records and not self._records[p].inputs \
                    and not self.get_children(p):
                self.remove_node(p)

    def update_node(self, name, updating_name):
        """`name` becomes `updating_name` (operation, flags, parents, observed data) while the
        children of `name` keep pointing at it; `updating_name` disappears."""
        incoming = self._records[updating_name]
        data = self._observed.pop(updating_name, None)
        old_inputs = self._records[name].inputs
        del self._records[updating_name]
        for other in self._records.values():      # nothing may keep pointing at the vanished name
            if updating_name in other.inputs:
                other.inputs = [p for p in other.inputs if p != updating_name]
        self._records[name] = incoming
        self._observed.pop(name, None)
        if data is not None:
            self._observed[name] = data
        for p in old_inputs:
            if p.startswith('_') and p in self._records and p not in incoming.inputs and \
                    not self._records[p].inputs and not self.get_children(p):
                self.remove_node(p)

    @property
    def parameter_names(self):
        return sorted(n for n, rec in self._records.items() if rec.has(PARAMETER))

    @parameter_names.setter
    def parameter_names(self, parameter_names):
        unknown = set(parameter_names) - set(self._records)
        if unknown:
            raise ValueError('Parameters {} not found from the model'.format(unknown))
        for n, rec in self._records.items():
            rec.set(PARAMETER, n in parameter_names)

    def copy(self):
        """A model with its own table and observed dict over the same operations / node state."""
        twin = ElfiModel(name='{}_copy_{}'.format(self.name, random_name()))
        twin._records = {n: rec.twin() for n, rec in self._records.items()}
        twin._observed = dict(self._observed)
        return twin

    def get_reference(self, name):
        return self._records[name].cls.reference(name, self)

    __getitem__ = get_reference

    def generate(self, batch_size=1, outputs=None, with_values=None, seed=None):
        """One batch of the named outputs (all nodes by default) as {name: array}."""
        if outputs is None:
            outputs = self.nodes
        elif isinstance(outputs, str):
            outputs = [outputs]
        if not isinstance(outputs, list):
            raise ValueError('Outputs must be a list of node names')
        context = ComputationContext(batch_size, seed='global' if seed is None else seed)
        return execute_batch(self, outputs, context, 0, with_values)


# ---------------------------------------------------------------------------- compile / run
def _constant_topological_order(nodes, successors):
    """The reference's deterministic order (elfi/executor.py:162-246): depth-first search from
    the alphabetically sorted nodes, children visited from the alphabetically last to the
    first, reverse finishing order.  `successors(node)` returns an iterable of children."""
    done, finishing = set(), []
    for start in sorted(nodes):
        if start in done:
            continue
        active = {start}
        trail = [(start, iter(sorted(successors(start), reverse=True)))]
        while trail:
            node, pending = trail[-1]
            nxt = next((c for c in pending if c not in done), None)
            if nxt is None:
                trail.pop()
                active.discard(node)
                done.add(node)
                finishing.append(node)
            elif nxt in active:
                raise ValueError('The model graph contains a cycle through {}'.format(nxt))
            else:
                active.add(nxt)
                trail.append((nxt, iter(sorted(successors(nxt), reverse=True))))
    finishing.reverse()
    return finishing


def _pack_observed(*twins):
    return tuple(twins)


class Step:
    """One node of a compiled plan: where its value comes from."""
    __slots__ = ('name', 'op', 'constant', 'args', 'kwargs', 'fuses_accept')

    def __init__(self, name, op=None, constant=_MISSING, fuses_accept=False):
        self.name = name
        self.op = op
        self.constant = constant
        self.args = []          # names, positional
        self.kwargs = {}        # keyword -> name
        self.fuses_accept = fuses_accept

    @property
    def sources(self):
        return self.args + list(self.kwargs.values())


class Plan:
    """A model lowered for a set of outputs: the steps the outputs depend on, in execution
    order."""

    def __init__(self, model_name, outputs, steps, order):
        self.model_name = model_name
        self.outputs = list(outputs)
        self.steps = steps                      # name -> Step
        self.order = order

    def has_node(self, name):
        return name in self.steps

    def __contains__(self, name):
        return name in self.steps

    def run(self, values, outputs, accept=None, keep_observed=None):
        """Evaluate `outputs` given the already known `values` (mutated); returns the extra
        products of fused steps as {('accepted', name): indices}."""
        pending, visit = set(), [o for o in outputs if o not in values]
        while visit:
            name = visit.pop()
            if name in pending or name in values:
                continue
            pending.add(name)
            visit.extend(self.steps[name].sources)
        extras = {}
        for name in self.order:
            if name not in pending:
                continue
            step = self.steps[name]
            if step.op is None:
                raise ValueError('Nothing provides a value for node {}'.format(name))
            kwargs = {k: values[src] for k, src in step.kwargs.items()}
            if accept is not None and step.fuses_accept and name in accept:
                kwargs['accept'] = accept[name]
            try:
                out = step.op(*[values[src] for src in step.args], **kwargs)
            except Exception as exc:
                note = "In executing node '{}': {}.".format(name, exc)
                try:
                    tagged = type(exc)(note)
                except Exception:                 # exception types with their own signature
                    tagged = RuntimeError(note)
                raise tagged.with_traceback(exc.__traceback__) from exc
            if isinstance(out, AcceptedOutput):
                extras[('accepted', name)] = out.accepted
                out = out.value
            values[name] = out
            if keep_observed is not None and is_observed_name(name):
                keep_observed[name] = out
        return extras


def compile_plan(model, outputs):
    """Lower `model` for `outputs` (node names, observed-twin names allowed).

    Every observable node X gets a twin ``_X_observed`` that applies X's operation to the
    twins of X's parents (a stochastic X -- a simulator -- has no inputs there: its twin is the
    observed data itself); a node that takes `observed=` gets a twin packing its parents' twins
    into a tuple.  Nodes flagged for batch size / meta / random state read the per-batch inputs
    of those names.  Only what the outputs depend on is kept."""
    table = model._records
    steps = {}
    for name, rec in table.items():
        if rec.constant is not _MISSING and rec.op is not None:
            raise ValueError("Cannot compile: node '{}' has both a value and an "
                             "operation".format(name))
        if rec.constant is _MISSING and rec.op is None:
            raise ValueError("Cannot compile: node '{}' has neither a value nor an "
                             "operation".format(name))
        step = steps[name] = Step(name, rec.op, rec.constant, rec.has(TAKES_ACCEPT))
        step.args = list(rec.inputs)
        if rec.has(TAKES_BATCH_SIZE):
            step.kwargs['batch_size'] = BATCH_SIZE_INPUT
        if rec.has(TAKES_META):
            step.kwargs['meta'] = META_INPUT
        if rec.has(STOCHASTIC):
            step.kwargs['random_state'] = RANDOM_STATE_INPUT

    def twin_or_self(parent):
        return observed_name(parent) if table[parent].has(OBSERVABLE) else parent

    for name, rec in table.items():
        if rec.has(OBSERVABLE):
            twin = steps[observed_name(name)] = Step(observed_name(name), rec.op, rec.constant)
        elif rec.has(TAKES_OBSERVED):
            twin = steps[observed_name(name)] = Step(observed_name(name), _pack_observed)
            steps[name].kwargs['observed'] = twin.name
        else:
            continue
        if not rec.has(STOCHASTIC):
            twin.args = [twin_or_self(p) for p in rec.inputs]
    for feed in (BATCH_SIZE_INPUT, META_INPUT, RANDOM_STATE_INPUT):
        if any(feed in s.kwargs.values() for s in steps.values()):
            steps[feed] = Step(feed)

    def upstream(roots):
        seen, visit = set(), list(roots)
        while visit:
            n = visit.pop()
            if n not in seen:
                seen.add(n)
                visit.extend(steps[n].sources)
        return seen

    for name, rec in table.items():
        if rec.has(TAKES_OBSERVED):
            for anc in upstream([observed_name(name)]):
                if anc in table and table[anc].has(STOCHASTIC):
                    raise ValueError('Observed nodes must be deterministic. Observed data '
                                     'depends on a non-deterministic node {}.'.format(anc))
    for o in outputs:
        if o not in steps:
            raise ValueError('Node {} is not in the model'.format(o))
    kept = upstream(outputs)
    steps = {n: s for n, s in steps.items() if n in kept}
    children = {n: [] for n in steps}
    for n, s in steps.items():
        for src in s.sources:
            children[src].append(n)
    order = _constant_topological_order(steps, children.__getitem__)
    return Plan(model.name, outputs, steps, order)


def _batch_random_state(context, batch_index):
    """The RandomState of one batch: numpy's global one for seed 'global', else a fresh one
    from the batch's sub seed (elfi/loader.py:131-178)."""
    seed = context.seed
    if isinstance(seed, str) and seed == 'global':
        return np.random.mtrand._rand
    if isinstance(seed, (int, np.integer)):
        sub = get_sub_seed(int(seed), batch_index, cache=context.caches.get('sub_seed'))
        return np.random.RandomState(sub)
    raise ValueError('Seed of type {} is not supported'.format(seed))


def execute_batch(model, outputs, context, batch_index, with_values=None, accept=None,
                  compiled=None):
    """Run one batch of `outputs`; returns {name: output}.

    `compiled` is the plan of a previous ``compile_plan(model, outputs)`` (samplers compile
    once per inference).  `accept` = {discrepancy name: thresholds} asks a device distance to
    also return the accepted row indices, found under the key ('accepted', name).

    Known before any step runs: observed data (-> twins of the nodes that carry it), the
    per-batch inputs, outputs already in the context's pool, `with_values`, constants, and --
    with a reused plan -- the observed twins evaluated by the first batch (they are
    deterministic functions of the observed data: checked at compile time; the reference
    re-evaluates them every batch, which here would be kernel launches and a D2H each)."""
    plan = compiled if compiled is not None else compile_plan(model, outputs)
    values = {}
    for name, data in model.observed.items():
        if observed_name(name) in plan:
            values[observed_name(name)] = data
    if BATCH_SIZE_INPUT in plan:
        values[BATCH_SIZE_INPUT] = context.batch_size
    if META_INPUT in plan:
        values[META_INPUT] = dict(batch_index=batch_index,
                                  submission_index=context.num_submissions,
                                  master_seed=context.seed, model_name=plan.model_name)
    if RANDOM_STATE_INPUT in plan:
        values[RANDOM_STATE_INPUT] = _batch_random_state(context, batch_index)
    wanted = list(plan.outputs)
    if context.pool is not None:
        # stored outputs replace their nodes; missing ones are requested so that the callback
        # can store them when the batch is done (elfi/loader.py:95-129)
        stored = context.pool.get_batch(batch_index)
        for name in context.pool.stores:
            if name in stored and name in plan:
                values[name] = stored[name]
            elif name in plan and name not in wanted:
                wanted.append(name)
    for name, val in (with_values or {}).items():
        if name in plan:
            values[name] = val
    for name, step in plan.steps.items():
        if step.constant is not _MISSING and name not in values:
            values[name] = step.constant
    twins = None
    if compiled is not None:
        twins = context.caches.setdefault('observed', {}).setdefault(id(plan), {})
        for name, val in twins.items():
            values.setdefault(name, val)
    extras = plan.run(values, wanted, accept=accept, keep_observed=twins)
    result = {name: values[name] for name in wanted}
    result.update(extras)
    return result


class AcceptedOutput:
    """Distance output + accepted row indices (fused acceptance)."""

    def __init__(self, value, accepted):
        self.value = value
        self.accepted = accepted


# ------------------------------------------------------------------------------------- nodes
class NodeReference:
    """A handle (model, name) on one row of a model's table.  Creating a node object inserts
    the row; ``model[name]`` re-creates a handle of the row's class."""

    # what a subclass contributes to its row
    _flags = 0

    def __init__(self, *parents, state=None, model=None, name=None):
        state = dict(state or {})
        if model is not None and not isinstance(model, ElfiModel):
            raise ValueError('Invalid model passed {}'.format(model))
        for p in parents:
            if isinstance(p, NodeReference):
                if model is None:
                    model = p.model
                elif p.model is not model:
                    raise ValueError('Parents are from different models!')
        self.model = get_default_model() if model is None else model
        self.name = self._resolve_name(name)
        record = NodeRecord(type(self), op=state.pop('op', None),
                            constant=state.pop('constant', _MISSING),
                            flags=self._flags | state.pop('flags', 0), attrs=state)
        self.model.insert(self.name, record)
        for p in parents:
            if not isinstance(p, NodeReference):     # plain values become hidden constants
                p = Constant(p, model=self.model, name='_' + self.name + '*')
            record.inputs.append(p.name)

    def _resolve_name(self, name):
        """An explicit name is used as is; 'base*' gets a random suffix; without a name a
        random one is made up (the reference reads the caller's assignment target instead)."""
        if name is not None and not name.endswith('*'):
            return name
        base = name[:-1] if name else '_' + type(self).__name__.lower()
        while True:
            candidate = '{}_{}'.format(base, random_name())
            if not self.model.has_node(candidate):
                return candidate

    @classmethod
    def reference(cls, name, model):
        handle = cls.__new__(cls)
        handle.name, handle.model = name, model
        return handle

    @property
    def record(self):
        if self.model is None:
            raise ValueError('{} {} is not initialized'.format(type(self).__name__, self.name))
        return self.model.record(self.name)

    @property
    def parents(self):
        return [self.model[p] for p in self.model.get_parents(self.name)]

    def become(self, other_node):
        """Replace this node by `other_node` in place: children keep their parent."""
        if other_node.model is not self.model:
            raise ValueError('The other node belongs to a different model')
        self.model.update_node(self.name, other_node.name)
        if not isinstance(self, self.record.cls):
            self.__class__ = self.record.cls
        other_node.name = self.name

    def generate(self, batch_size=1, with_values=None):
        return self.model.generate(batch_size, self.name, with_values=with_values)[self.name]

    @property
    def uses_meta(self):
        return self.record.has(TAKES_META)

    @uses_meta.setter
    def uses_meta(self, on):
        self.record.set(TAKES_META, bool(on))

    def __repr__(self):
        return "{}(name='{}')".format(type(self).__name__, self.name)

    def __str__(self):
        return self.name


class Constant(NodeReference):
    def __init__(self, value, **kwargs):
        super().__init__(state=dict(constant=value), **kwargs)


class _HostOperation:
    """User-supplied Operation callables expect NumPy: device inputs are copied to the host
    first (explicit D2H; generic Operations are host logic, not part of the CUDA hot path)."""

    def __init__(self, fn):
        self.fn = fn

    def __call__(self, *args, **kwargs):
        args = [dev.to_host(a) if dev.is_device_array(a) else a for a in args]
        kwargs = {k: (dev.to_host(v) if dev.is_device_array(v) else v) for k, v in kwargs.items()}
        return self.fn(*args, **kwargs)


class Operation(NodeReference):
    def __init__(self, fn, *parents, **kwargs):
        super().__init__(*parents, state=dict(op=_HostOperation(fn)), **kwargs)


def _draw(*params, batch_size, distribution, size=None, random_state=None):
    """One batch of a random variable: `size` is the shape of a single draw."""
    shape = (batch_size,) + (size or ())
    return distribution.rvs(*params, size=shape, random_state=random_state)


class RandomVariable(NodeReference):
    """`distribution` is a scipy.stats name or any object with ``rvs(*params, size,
    random_state)``."""
    _flags = STOCHASTIC | TAKES_BATCH_SIZE

    def __init__(self, distribution, *params, size=None, **kwargs):
        if size is not None and not isinstance(size, tuple):
            size = (size,)
        dist = scipy_from_str(distribution) if isinstance(distribution, str) else distribution
        if not hasattr(dist, 'rvs'):
            raise ValueError('Distribution {} must implement a rvs method'.format(distribution))
        state = dict(op=partial(_draw, distribution=dist, size=size), distribution=distribution,
                     size=size)
        super().__init__(*params, state=state, **kwargs)

    @property
    def distribution(self):
        dist = self.record.attrs['distribution']
        return scipy_from_str(dist) if isinstance(dist, str) else dist

    @property
    def size(self):
        return self.record.attrs['size']


class Prior(RandomVariable):
    _flags = RandomVariable._flags | PARAMETER


class _Observable(NodeReference):
    _flags = OBSERVABLE

    def _set_observed(self, observed):
        if observed is not None:
            self.model.observed[self.name] = observed

    @property
    def observed(self):
        twin = observed_name(self.name)
        return self.model.generate(0, twin)[twin]


class Simulator(_Observable):
    """fn(*params, batch_size, random_state) -> array of length batch_size."""
    _flags = OBSERVABLE | STOCHASTIC | TAKES_BATCH_SIZE

    def __init__(self, fn, *params, observed=None, **kwargs):
        super().__init__(*params, state=dict(op=fn), **kwargs)
        self._set_observed(observed)


def _require_parents(parents):
    if not parents:
        raise ValueError('This node requires that at least one parent is specified.')


class Summary(_Observable):
    """fn(*parents) -> summary statistic; may return a device array."""

    def __init__(self, fn, *parents, observed=None, **kwargs):
        _require_parents(parents)
        super().__init__(*parents, state=dict(op=fn), **kwargs)
        self._set_observed(observed)


class Discrepancy(NodeReference):
    """discrepancy(*summaries, observed=tuple) -> (B,) or (B, K)."""
    _flags = TAKES_OBSERVED

    def __init__(self, discrepancy, *parents, **kwargs):
        _require_parents(parents)
        state = dict(kwargs.pop('state', None) or {}, op=discrepancy)
        super().__init__(*parents, state=state, **kwargs)


def _stack_summaries(summaries):
    """np.column_stack(summaries) of elfi/model/utils.py:39 as a device matrix.
    A single 2-d parent is used in place (no copy); lazy simulator output is materialised."""
    import torch
    cols = []
    for s in summaries:
        if isinstance(s, LazySimulation):
            s = s.materialize()
        t = s if dev.is_device_array(s) else dev.to_device(np.asarray(s, dtype=np.float64))
        if t.dim() > 2:
            raise ValueError('Incompatible data shape for the distance node. Please check '
                             'summary (XA) and observed (XB) output data dimensions. They '
                             'have to be at most 2d.')
        cols.append(t if t.dim() == 2 else t[:, None])
    if len(cols) == 1:
        return cols[0]
    # columns that are adjacent views of one row-major matrix (e.g. the (B, 2) output of the fused
    # MA2 summaries) are re-assembled without a copy
    width = sum(c.shape[1] for c in cols)
    first = cols[0]
    if first.stride(0) == width and all(
            c.stride(0) == width and (c.shape[1] == 1 or c.stride(1) == 1) and
            c.data_ptr() == first.data_ptr() + 8 * sum(x.shape[1] for x in cols[:k]) and
            c.shape[0] == first.shape[0] for k, c in enumerate(cols)):
        return torch.as_strided(first, (first.shape[0], width), (width, 1))
    return torch.cat(cols, dim=1)


_OBSERVED_ROWS = {}     # id(observed tuple) -> [the tuple, stacked host row, its device twin]


def _stack_observed(observed):
    """The observed summaries as one (1, D) host row; one D2H per inference, not per batch."""
    hit = _OBSERVED_ROWS.get(id(observed))
    if hit is not None and hit[0] is observed:
        return hit[1]
    obs = [np.atleast_2d(dev.to_host(o)) for o in observed]
    row = np.concatenate(obs, axis=1).astype(np.float64)
    if len(_OBSERVED_ROWS) > 64:
        _OBSERVED_ROWS.clear()
    _OBSERVED_ROWS[id(observed)] = [observed, row, None]
    return row


def _observed_on_device(observed):
    """Device twin of :func:`_stack_observed` (a pageable H2D copy synchronises the stream: made
    once per inference, the distance kernels of all batches read the same D doubles)."""
    row = _stack_observed(observed)
    hit = _OBSERVED_ROWS[id(observed)]
    if hit[2] is None:
        hit[2] = dev.to_device(row.ravel())
    return hit[2]


_DEVICE_CONSTANTS = {}  # id(host array) -> (the array, device twin): operator constants (w, V)


def _device_constant(arr):
    """Device twin of a host array that an operator was constructed with (cdist's w / V): copied
    once, not with every batch (each pageable H2D copy synchronises the stream)."""
    if arr is None or dev.is_device_array(arr):
        return arr
    hit = _DEVICE_CONSTANTS.get(id(arr))
    if hit is not None and hit[0] is arr:
        return hit[1]
    if len(_DEVICE_CONSTANTS) > 64:
        _DEVICE_CONSTANTS.clear()
    twin = dev.to_device(np.asarray(arr, dtype=np.float64))
    _DEVICE_CONSTANTS[id(arr)] = (arr, twin)
    return twin


def device_euclidean_discrepancy(*summaries, observed, w=None, accept=None):
    """distance_as_discrepancy (elfi/model/utils.py:37-52) for the Euclidean family, on device.
    The unweighted distance of lazy simulator output that offers a fused one is computed in the
    simulator kernel, without writing the data."""
    if w is None and len(summaries) == 1 and isinstance(summaries[0], LazySimulation) and \
            summaries[0].euclidean is not None:
        if _stack_observed(observed).shape[0] != 1:
            raise ValueError('observed summaries must form a single row')
        d, idx = summaries[0].euclidean(_observed_on_device(observed), accept)
        return AcceptedOutput(d, idx) if accept is not None else d
    X = _stack_summaries(summaries)
    if _stack_observed(observed).shape[0] != 1:
        raise ValueError('observed summaries must form a single row')
    d, idx = ops.dist_euclid(X, _observed_on_device(observed), w=_device_constant(w),
                             thresholds=accept)
    return AcceptedOutput(d, idx) if accept is not None else d


DEVICE_METRICS = ('sqeuclidean', 'cityblock', 'chebyshev', 'minkowski')


def device_metric_discrepancy(metric, *summaries, observed, p=2.0, accept=None):
    """distance_as_discrepancy for the other unweighted cdist metrics that have a kernel."""
    X = _stack_summaries(summaries)
    if _stack_observed(observed).shape[0] != 1:
        raise ValueError('observed summaries must form a single row')
    thr = None if accept is None else np.atleast_1d(dev.to_host(accept))
    d, idx = ops.dist_metric(X, _observed_on_device(observed), metric, p=p, threshold=thr)
    return AcceptedOutput(d, idx) if accept is not None else d


def device_seuclidean_discrepancy(*summaries, observed, V, accept=None):
    """distance_as_discrepancy for cdist's 'seuclidean' (V = component variances)."""
    X = _stack_summaries(summaries)
    if _stack_observed(observed).shape[0] != 1:
        raise ValueError('observed summaries must form a single row')
    thr = None if accept is None else np.atleast_1d(dev.to_host(accept))
    d, idx = ops.dist_seuclidean(X, _observed_on_device(observed), _device_constant(V),
                                 threshold=thr)
    return AcceptedOutput(d, idx) if accept is not None else d


def device_mahalanobis_discrepancy(*summaries, observed, VI, accept=None):
    """distance_as_discrepancy for cdist's 'mahalanobis' (VI = inverse covariance matrix)."""
    X = _stack_summaries(summaries)
    if _stack_observed(observed).shape[0] != 1:
        raise ValueError('observed summaries must form a single row')
    thr = None if accept is None else np.atleast_1d(dev.to_host(accept))
    d, idx = ops.dist_mahalanobis(X, _observed_on_device(observed), _device_constant(VI),
                                  threshold=thr)
    return AcceptedOutput(d, idx) if accept is not None else d


def host_distance_as_discrepancy(dist, *summaries, observed):
    """Generic path for metrics without a CUDA kernel: explicit error, never a silent fallback."""
    raise NotImplementedError(
        "elfi_b200.Distance implements the Euclidean family on the device "
        "('euclidean' with or without w=, 'seuclidean' with V=), 'mahalanobis' with VI= and "
        "'sqeuclidean', 'cityblock', "
        "'chebyshev', 'minkowski' (p=) unweighted. Metric {!r} with these keywords has no "
        "CUDA kernel; use elfi_b200.Discrepancy with your own callable.".format(dist))


_REQUIRED_METRIC_KEYWORD = {'wminkowski': 'w', 'seuclidean': 'V', 'mahalanobis': 'VI'}


def _device_metric_operation(metric, kw):
    """The device operation for cdist metric `metric` with cdist keywords `kw`, or None when no
    kernel computes that combination."""
    given = set(kw)
    if metric == 'euclidean' and given <= {'w'}:
        return partial(device_euclidean_discrepancy, w=kw.get('w'))
    if metric == 'seuclidean' and given == {'V'}:
        return partial(device_seuclidean_discrepancy, V=np.asarray(kw['V'], dtype=np.float64))
    if metric == 'mahalanobis' and given == {'VI'}:
        return partial(device_mahalanobis_discrepancy,
                       VI=np.asarray(kw['VI'], dtype=np.float64))
    if metric == 'minkowski' and given <= {'p'}:
        return partial(device_metric_discrepancy, metric, p=kw.get('p', 2.0))
    if metric in DEVICE_METRICS and not given:
        return partial(device_metric_discrepancy, metric)
    return None


class Distance(Discrepancy):
    """Distance(metric, *summaries[, p=, w=, V=, VI=]): a cdist metric name (device kernel, fused
    acceptance) or a callable ``f(XA, XB)`` (host operation).  Node semantics of
    elfi/model/elfi_model.py:974-1044."""

    def __init__(self, distance, *summaries, **kwargs):
        _require_parents(summaries)
        state = {}
        if callable(distance):
            def op(*summaries, observed, _f=distance):
                d = _f(_stack_summaries(summaries), _stack_observed(observed))
                return d.reshape(-1) if d.ndim == 2 and d.shape[1] == 1 else d
        else:
            need = _REQUIRED_METRIC_KEYWORD.get(distance)
            if need is not None and need not in kwargs:
                raise ValueError('Parameter {} must be specified for distance={}.'.format(
                    need, distance))
            kw = {k: kwargs.pop(k) for k in ('p', 'w', 'V', 'VI') if k in kwargs}
            op = _device_metric_operation(distance, kw)
            if op is None:
                op = partial(host_distance_as_discrepancy, distance)
            else:
                state['flags'] = TAKES_ACCEPT
        super().__init__(op, *summaries, state=state, **kwargs)
        self.record.attrs['distance'] = distance


class AdaptiveDistance(Discrepancy):
    """Euclidean distance with adaptive per-summary scale (Prangle 2017);
    elfi/model/elfi_model.py:1047-1151.  State: w (list of weight vectors, first None),
    store = [n, mean, M2] merged batch by batch from device column moments."""

    def __init__(self, *summaries, **kwargs):
        _require_parents(summaries)
        state = dict(flags=TAKES_ACCEPT)
        super().__init__(self._nested_discrepancy, *summaries, state=state, **kwargs)
        self.init_state()

    # the operation is a bound method of a reference; look the state up at call time
    def _nested_discrepancy(self, *summaries, observed, accept=None):
        X = _stack_summaries(summaries)
        ws = self._s['w']
        D = X.shape[1]
        key = tuple(id(w) for w in ws)       # (K, D) squared weights: rebuilt when a round is added
        held = self._s.get('_W_dev')
        if held is None or held[0] != key or held[1].shape[1] != D:
            W = np.stack([np.ones(D) if w is None else np.asarray(w, dtype=np.float64) ** 2
                          for w in ws])
            held = self._s['_W_dev'] = (key, dev.to_device(W))
        # the batch's column moments come out of the same read of X; add_data picks them up
        d, idx, mom = ops.dist_euclid(X, _observed_on_device(observed), w=held[1],
                                      thresholds=accept, moments=True)
        self._s['_batch_moments'] = (X, mom)
        return AcceptedOutput(d, idx) if accept is not None else d

    @property
    def _s(self):
        return self.record.attrs

    def init_state(self):
        self._s['w'] = [None]
        self._s['store'] = 3 * [None]
        self.init_adaptation_round()

    def init_adaptation_round(self):
        if 'store' not in self._s:
            self.init_state()
        self._s['store'] = [0, 0, 0]
        self._s.pop('_batch_moments', None)

    def add_data(self, *data):
        """Chan-merge this batch's device column moments into (n, mean, M2); algebraically the
        batch Welford update of elfi_model.py:1117-1123."""
        X = _stack_summaries(data)
        nb = X.shape[0]
        held = self._s.pop('_batch_moments', None)
        if held is not None and held[0].data_ptr() == X.data_ptr() and \
                held[0].shape == X.shape and held[0].stride() == X.stride():
            mean_b, m2_b = held[1].cpu().numpy()      # fused with the distance pass
        else:
            mean_b, m2_b = ops.colmoments(X)
        n0, m0, s0 = self._s['store']
        n1 = n0 + nb
        delta = mean_b - m0
        self._s['store'] = [n1, m0 + delta * (nb / n1), s0 + m2_b + delta ** 2 * (n0 * nb / n1)]
        self._s['scale'] = np.sqrt(self._s['store'][2] / n1)

    def update_distance(self):
        weis = 1 / self._s['scale']
        self._s['w'].append(weis)
        self.init_adaptation_round()

    def nested_distance(self, u, v):
        return self._nested_discrepancy(u, observed=(v,))
