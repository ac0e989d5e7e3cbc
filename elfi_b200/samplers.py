"""Rejection / SMC-ABC samplers with the population arithmetic on the device.

Host control flow mirrors the reference (file:line in elfi-dev/elfi):
  ParameterInference.infer/iterate      elfi/methods/inference/parameter_inference.py:226-305
  Rejection                             elfi/methods/inference/samplers.py:57-317
  SMC                                   elfi/methods/inference/samplers.py:320-559
  AdaptiveDistanceSMC                   elfi/methods/inference/samplers.py:562-659
  ModelPrior.logpdf                     elfi/model/extensions.py:120-211
  GMDistribution.rvs / logpdf           elfi/methods/utils.py:142-272
What moved to the GPU: summaries + distances (+ acceptance) per batch, the running top-n merge
(sort + gather instead of argsort + fancy indexing over n + batch_size rows), the weighted
quantile, the O(N^2) proposal density, importance weights and weighted variance.

Multi-GPU (one process per GPU, torch.distributed): batch index b is computed by rank
b % world_size; ranks keep local top-n states and exchange them with ONE all-gather when a
population is extracted (fixed capacity n rows per rank), after which every rank holds the same
population.  The O(N^2) density is sharded over the new particles and all-gathered.
"""
import logging
from functools import reduce
from math import ceil
from operator import add

import numpy as np
import scipy.stats as ss
import torch

from . import device as dev
from . import model as em
from . import ops
from . import sharding
from .results import DeviceOutputs, Sample, SmcSample
from .throughput import LazySimulation

logger = logging.getLogger(__name__)


class _PhaseTimer:
    """Optional wall-clock phase accounting (ELFI_B200_TIMING=1): synchronises the device at
    phase boundaries, so it is off by default."""

    def __init__(self):
        import os
        self.on = os.environ.get('ELFI_B200_TIMING') == '1'
        self.tot = {}

    def __call__(self, name):
        timer = self

        class _Ctx:
            def __enter__(self_inner):
                if timer.on:
                    torch.cuda.synchronize()
                    import time
                    self_inner.t0 = time.perf_counter()

            def __exit__(self_inner, *a):
                if timer.on:
                    torch.cuda.synchronize()
                    import time
                    timer.tot[name] = timer.tot.get(name, 0.0) + time.perf_counter() - self_inner.t0
        return _Ctx()

    def report(self):
        return {k: round(v, 4) for k, v in sorted(self.tot.items(), key=lambda kv: -kv[1])}


PHASES = _PhaseTimer()

__all__ = ['Rejection', 'SMC', 'AdaptiveDistanceSMC', 'AdaptiveThresholdSMC', 'ModelPrior',
           'GMDistribution', 'DensityRatioEstimation']


# ----------------------------------------------------------------------------- communication
COMM_STATS = {'all_gather_calls': 0, 'all_gather_bytes': 0}   # data-path collectives (received bytes)


class Comm:
    """torch.distributed plumbing (NCCL on GPUs, gloo in CPU tests); identity when single."""

    def __init__(self, enabled=True):
        import torch.distributed as dist
        self.dist = dist
        self.on = bool(enabled) and dist.is_available() and dist.is_initialized() \
            and dist.get_world_size() > 1
        self.rank = dist.get_rank() if self.on else 0
        self.size = dist.get_world_size() if self.on else 1

    def all_gather_rows(self, t):
        """Concatenate equally shaped tensors of all ranks along axis 0 (rank order)."""
        if not self.on:
            return t
        t = t.contiguous()
        out = torch.empty((self.size * t.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype,
                          device=t.device)
        self.dist.all_gather_into_tensor(out, t)
        COMM_STATS['all_gather_calls'] += 1
        COMM_STATS['all_gather_bytes'] += out.numel() * out.element_size()
        return out

    def all_gather_ints(self, values):
        """Every rank's list of integers as a (size, len(values)) int64 host array: ONE small
        collective for all the per-rank counters a step needs (counts, n_sim, n_batches)."""
        vals = np.asarray(values, dtype=np.int64).reshape(1, -1)
        if not self.on:
            return vals
        devname = 'cuda' if self.dist.get_backend() == 'nccl' else 'cpu'
        t = torch.from_numpy(vals).to(devname)
        out = torch.empty((self.size, vals.shape[1]), dtype=torch.int64, device=devname)
        self.dist.all_gather_into_tensor(out, t)
        return out.cpu().numpy()

    def all_reduce_sum(self, value):
        if not self.on:
            return value
        backend = self.dist.get_backend()
        devname = 'cuda' if backend == 'nccl' else 'cpu'
        t = torch.tensor([float(value)], dtype=torch.float64, device=devname)
        self.dist.all_reduce(t)
        return float(t.item())


# -------------------------------------------------------------------------------- prior, GM
def numgrad(fn, x, h=None, replace_neg_inf=True):
    """Central-difference gradient of a scalar function at one point
    (elfi/methods/utils.py:275-314): the 3 * dim points x + (-1, 0, 1) h e_i go to `fn` in one
    call; if any value is -inf (a log density outside its support) the gradient is zero."""
    h = np.asanyarray(0.00001 if h is None else h, dtype=float).reshape(-1)
    x = np.asanyarray(x, dtype=float).reshape(-1)
    dim = len(x)
    offsets = (np.arange(3) - 1.0)[:, None, None] * (np.eye(dim) * h)[None, :, :]
    f = np.asarray(fn((x + offsets).reshape(3 * dim, dim))).reshape((3, dim))
    if replace_neg_inf and np.any(np.isneginf(f)):
        return np.zeros(dim)
    return np.gradient(f, *h, axis=0)[1, :]


def resolve_sigmas(parameter_names, sigma_proposals=None, bounds=None):
    """Proposal standard deviations in parameter order (elfi/methods/utils.py:460-503): a dict
    keyed by parameter name, or by default a tenth of each bound interval."""
    if sigma_proposals is None:
        return [(hi - lo) / 10 for lo, hi in bounds]
    if isinstance(sigma_proposals, dict):
        if set(sigma_proposals) != set(parameter_names):
            raise ValueError("sigma_proposals' keys have to be identical to "
                             "target_model.parameter_names.")
        return [sigma_proposals[name] for name in parameter_names]
    raise ValueError("If provided, sigma_proposals need to be input as a dict.")


class ModelPrior:
    """Joint prior of the model parameters (elfi/model/extensions.py:120-245): logpdf is the sum
    of each parameter node's distribution.logpdf(x_node, *parent values), evaluated through the
    graph so conditional priors (MA2's t2 | t1) work.  Host side: priors are arbitrary Python."""

    def __init__(self, model, parameter_names=None):
        model = model.copy()
        self.parameter_names = parameter_names or model.parameter_names
        for p in self.parameter_names:
            if p not in model.parameter_names:
                raise ValueError("Parameter '{}' not found in model parameters.".format(p))
        self.dim = len(self.parameter_names)
        self._model = model
        self._nets = {}
        for log in (False, True):
            attr = 'logpdf' if log else 'pdf'
            nodes = []
            for n in model.parameter_names:
                node = model[n]
                op = getattr(node.distribution, attr)
                nodes.append(em.Operation(op, node, *node.parents, model=model,
                                          name='_{}_{}'.format(n, attr)))
            combine = add if log else (lambda a, b: a * b)
            joint = em.Operation(lambda *a, _c=combine: reduce(_c, a), *nodes, model=model,
                                 name='_joint_{}*'.format(attr))
            self._nets[log] = (joint.name, em.compile_plan(model, [joint.name]))

    def _evaluate(self, x, log):
        x = np.asanyarray(x)
        ndim = x.ndim
        x = x.reshape((-1, self.dim))
        name, net = self._nets[log]
        context = em.ComputationContext(len(x), seed=0)
        batch = {p: x[:, i] for i, p in enumerate(self.parameter_names)}
        val = em.execute_batch(self._model, [name], context, 0, with_values=batch,
                               compiled=net)[name]
        if ndim == 0 or (ndim == 1 and self.dim > 1):
            val = val[0]
        return val

    def pdf(self, x):
        return self._evaluate(x, False)

    def logpdf(self, x):
        return self._evaluate(x, True)

    def gradient_logpdf(self, x, stepsize=None):
        """Central-difference gradient of the joint log prior, row by row; zero where it is not
        finite, e.g. outside the support (elfi/model/extensions.py:217-242)."""
        x = np.asanyarray(x, dtype=float)
        ndim = x.ndim
        x = x.reshape((-1, self.dim))
        # numgrad for every row, with all 3 * dim * len(x) probe points in one logpdf call
        h = np.asanyarray(0.00001 if stepsize is None else stepsize, dtype=float).reshape(-1)
        offsets = (np.arange(3) - 1.0)[:, None, None] * (np.eye(self.dim) * h)[None, :, :]
        probes = x[:, None, None, :] + offsets[None, :, :, :]          # (n, 3, dim, dim)
        f = np.asarray(self.logpdf(probes.reshape(-1, self.dim))).reshape(len(x), 3, self.dim)
        with np.errstate(invalid='ignore'):               # -inf probes are zeroed below
            grads = np.gradient(f, *h, axis=1)[:, 1, :]
        grads[np.any(np.isneginf(f), axis=(1, 2))] = 0    # a probe outside the support
        grads[~np.isfinite(grads)] = 0
        if ndim == 0 or (ndim == 1 and self.dim > 1):
            grads = grads[0]
        return grads

    def rvs(self, size=None, random_state=None):
        random_state = np.random if random_state is None else random_state
        context = em.ComputationContext(size or 1, seed='global')
        batch = em.execute_batch(self._model, list(self.parameter_names), context, 0,
                                 with_values={'_random_state': random_state})
        rvs = np.column_stack([dev.to_host(batch[p]) for p in self.parameter_names])
        if self.dim == 1:
            rvs = rvs.reshape(size or 1)
        return rvs[0] if size is None else rvs


def normalize_weights(weights):
    """elfi/methods/utils.py:80-88."""
    w = np.atleast_1d(weights)
    total = np.sum(weights)
    if (w < 0).any() or total == 0:
        raise ValueError('Weights must be non-negative and not all zero')
    return w / total


class GMDistribution:
    """Gaussian mixture with shared covariance (elfi/methods/utils.py:142-272).
    logpdf/pdf run on the device; rvs consumes the host RandomState like the reference."""

    @classmethod
    def logpdf(cls, x, means, cov=1, weights=None):
        return ops.gm_logpdf(x, means, cov, weights)

    @classmethod
    def pdf(cls, x, means, cov=1, weights=None):
        return torch.exp(ops.gm_logpdf(x, means, cov, weights))

    @classmethod
    def rvs(cls, means, cov=1, weights=None, size=1, prior_logpdf=None, random_state=None):
        random_state = random_state or np.random
        means = np.atleast_1d(np.squeeze(means))
        if means.ndim > 2:
            raise ValueError('means.ndim = {} but must be at most 2.'.format(means.ndim))
        if weights is None:
            weights = np.ones(len(means))
        weights = normalize_weights(weights)
        no_wrap = size is None
        if no_wrap:
            size = 1
        output = np.empty((size,) + means.shape[1:])
        n_accepted, n_left, trials = 0, size, 0
        while n_accepted < size:
            inds = random_state.choice(len(means), size=n_left, p=weights)
            centres = means[inds]
            perturb = ss.multivariate_normal.rvs(mean=means[0] * 0, cov=cov,
                                                 random_state=random_state, size=n_left)
            x = centres + perturb
            if prior_logpdf is not None:
                x = x[np.isfinite(prior_logpdf(x))]
            k = len(x)
            output[n_accepted:n_accepted + k] = x
            n_accepted += k
            n_left -= k
            trials += 1
            if trials == 100:
                logger.warning("SMC: It appears to be difficult to find enough valid proposals "
                               "with prior pdf > 0. ELFI will keep trying, but you may wish "
                               "to kill the process and adjust the model priors.")
        return output[0] if no_wrap else output


# ----------------------------------------------------------------------------- base class
class ParameterInference:
    """Batch loop of elfi's ParameterInference for a single in-order device client."""

    def __init__(self, model, output_names, batch_size=1, seed=None, pool=None,
                 max_parallel_batches=None, distributed=True):
        """`distributed=False` keeps the inference on this rank only even when a
        torch.distributed process group is initialised."""
        model = model.model if isinstance(model, em.NodeReference) else model
        if not model.parameter_names:
            raise ValueError('Model {} defines no parameters'.format(model))
        self.model = model.copy()
        self.output_names = self._check_outputs(output_names)
        self.computation_context = em.ComputationContext(batch_size=batch_size, seed=seed,
                                                         pool=pool)
        self._compiled = em.compile_plan(self.model, self.output_names)
        self._distributed = distributed
        self.comm = Comm(distributed)
        self.max_parallel_batches = max_parallel_batches or self.comm.size
        if self.max_parallel_batches <= 0:
            raise ValueError('Value for max_parallel_batches ({}) must be at least one.'.format(
                self.max_parallel_batches))
        # Batches are processed in groups: `world_size` batches per step across the ranks
        # (batch b on rank b % world_size), or `max_parallel_batches` consecutive batches on a
        # single rank -- the reference keeps that many batches in flight
        # (parameter_inference.py:270-305).  Objectives are re-estimated and `finished` is tested
        # at group boundaries only, so a W-rank run and a single-rank run with
        # max_parallel_batches=W process exactly the same batches.
        self._group = 1 if self.comm.on else int(self.max_parallel_batches)
        self.state = dict(n_sim=0, n_batches=0)
        self.objective = dict()
        self._next_batch_index = 0

    @property
    def seed(self):
        return self.computation_context.seed

    @property
    def pool(self):
        """The output pool of the inference (parameter_inference.py:111-114)."""
        return self.computation_context.pool

    @property
    def parameter_names(self):
        return self.model.parameter_names

    @property
    def batch_size(self):
        return self.computation_context.batch_size

    def set_objective(self, *args, **kwargs):
        raise NotImplementedError

    def extract_result(self):
        raise NotImplementedError

    def update(self, batch, batch_index):
        self.state['n_batches'] += 1
        self.state['n_sim'] += self.batch_size

    def prepare_new_batch(self, batch_index):
        pass

    def _accept_hint(self):
        return None

    def _run_batch(self, batch_index, values):
        batch = em.execute_batch(self.model, self.output_names, self.computation_context,
                                 batch_index, with_values=values, accept=self._accept_hint(),
                                 compiled=self._compiled)
        self.computation_context.num_submissions += 1
        self.computation_context.callback(batch, batch_index)
        return batch

    def infer(self, *args, vis=None, bar=True, **kwargs):
        self.set_objective(*args, **kwargs)
        while not self.finished:
            self.iterate()
        return self.extract_result()

    def iterate(self):
        """One batch: prepare -> execute on the device -> update (in batch_index order)."""
        batch_index = self._next_batch_index
        with PHASES('prepare_new_batch'):
            values = self.prepare_new_batch(batch_index)
        self._next_batch_index += 1
        with PHASES('run_batch'):
            batch = self._run_batch(batch_index, values)
        with PHASES('update'):
            self.update(batch, batch_index)

    @property
    def finished(self):
        if self.state['n_batches'] % self._group:
            return False
        return self._objective_n_batches <= self.state['n_batches']

    def _round_up_to_group(self, n_batches):
        g = self._group
        return int(ceil(n_batches / g)) * g if g > 1 else n_batches

    @property
    def _objective_n_batches(self):
        if 'n_batches' in self.objective:
            return self.objective['n_batches']
        if 'n_sim' in self.objective:
            return ceil(self.objective['n_sim'] / self.batch_size)
        raise ValueError('Objective must define either `n_batches` or `n_sim`.')

    def _extract_result_kwargs(self):
        return {'method_name': self.__class__.__name__, 'parameter_names': self.parameter_names,
                'seed': self.seed, 'n_sim': self.state['n_sim'],
                'n_batches': self.state['n_batches']}

    @staticmethod
    def _resolve_model(model, target, default_reference_class=em.NodeReference):
        """(model, target node name) from either (node, anything) or (model, node or name)."""
        if isinstance(model, em.NodeReference):
            model, target = model.model, model
        elif target is None:
            raise NotImplementedError('{}: the target node must be named when a model is '
                                      'given'.format(model))
        node = model[target] if isinstance(target, str) else target
        if not isinstance(node, default_reference_class):
            raise ValueError('{!r} is not a {}'.format(node, default_reference_class.__name__))
        return model, node.name

    def _check_outputs(self, output_names):
        """Node names (handles are accepted) in first-mention order, each once, all in the
        model."""
        names = [n.name if isinstance(n, em.NodeReference) else n for n in output_names or []]
        for name in names:
            if not isinstance(name, str):
                raise ValueError('Outputs are named by strings; got {!r}'.format(name))
            if not self.model.has_node(name):
                raise ValueError('Requested output {} is not a node of the model'.format(name))
        return list(dict.fromkeys(names))


class Sampler(ParameterInference):
    def sample(self, n_samples, *args, **kwargs):
        bar = kwargs.pop('bar', True)
        self.bar = bar
        return self.infer(n_samples, *args, bar=bar, **kwargs)

    def _extract_result_kwargs(self):
        kwargs = super()._extract_result_kwargs()
        for key in ['threshold', 'accept_rate']:
            if key in self.state:
                kwargs[key] = self.state[key]
        if hasattr(self, 'discrepancy_name'):
            kwargs['discrepancy_name'] = self.discrepancy_name
        return kwargs


# ------------------------------------------------------------------------------- rejection
def _batch_key(seed, batch_index):
    """Philox key of one batch's device proposals: splitmix64 of (round seed, batch index)."""
    m = (1 << 64) - 1
    z = (int(seed) * 0x9E3779B97F4A7C15 + int(batch_index) + 1) & m
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & m
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & m
    return int((z ^ (z >> 31)) & ((1 << 63) - 1))


def _to_dev_f64(x):
    if isinstance(x, LazySimulation):     # a simulator output kept in a sample: its data
        return x.materialize()
    return x if dev.is_device_array(x) else dev.to_device(np.asarray(x, dtype=np.float64))


class Rejection(Sampler):
    """Parallel ABC rejection sampler; the running best-n state lives on the device."""

    def __init__(self, model, discrepancy_name=None, output_names=None, **kwargs):
        model, discrepancy_name = self._resolve_model(model, discrepancy_name)
        # outputs the caller asked for by name travel in full in every multi-rank exchange; the
        # summaries an adaptive distance adds for its own re-scoring stay sharded (see
        # _gather_ranks_adaptive)
        self._full_exchange = set(n.name if isinstance(n, em.NodeReference) else n
                                  for n in (output_names or []))
        output_names = [discrepancy_name] + model.parameter_names + (output_names or [])
        self.adaptive = isinstance(model[discrepancy_name], em.AdaptiveDistance)
        if self.adaptive:
            model[discrepancy_name].init_adaptation_round()
            self.sums = [s.name for s in model[discrepancy_name].parents]
            for k in self.sums:
                if k not in output_names:
                    output_names.append(k)
        super().__init__(model, output_names, **kwargs)
        self.discrepancy_name = discrepancy_name

    def set_objective(self, n_samples, threshold=None, quantile=None, n_sim=None):
        if quantile is None and threshold is None and n_sim is None:
            quantile = .01
        self.state = dict(samples=None, threshold=np.inf, n_sim=0, accept_rate=1, n_batches=0)
        if quantile:
            n_sim = ceil(n_samples / quantile)
        if n_sim:
            n_batches = ceil(n_sim / self.batch_size)
            if self.comm.on:
                n_batches = sharding.batches_per_rank(n_batches, self.comm.size)
            n_batches = self._round_up_to_group(n_batches)
        else:
            n_batches = 1 if self.comm.on else self.max_parallel_batches
        self.objective = dict(n_samples=n_samples, threshold=threshold, n_batches=n_batches)
        self._next_batch_index = 0
        self._n_acceptable = 0
        self._n_valid = 0          # filled rows of the local best-n buffers
        self._gathered = False     # multi-rank: the ranks' buffers have been merged

    # -- device-side acceptance: thresholds are handed to the distance kernel
    def _accept_hint(self):
        thr = self.objective.get('threshold')
        if thr is None:
            # quantile / n_sim mode: every row of the batch is a candidate, as in the reference
            # (samplers.py:219-221).  Pruning with the buffer's current n-th distance would shrink
            # the merge sort, but the accepted COUNT then sizes the merge and costs one host round
            # trip per batch (more than the extra sort work costs: the radix passes are latency
            # bound at these sizes); without it nothing in this
            # mode waits for the device until the result is extracted.
            return None
        return {self.discrepancy_name: np.atleast_1d(np.asarray(thr, dtype=np.float64))}

    def update(self, batch, batch_index):
        if self._gathered:
            raise RuntimeError('the local best-n buffers were already merged across the ranks; '
                               'call set_objective() before simulating further batches')
        super().update(batch, batch_index)
        if self.state['samples'] is None:
            self._init_samples_lazy(batch)
        self._merge_batch(batch)
        if self.state['n_batches'] % self._group == 0:
            self._update_objective_n_batches()     # threshold mode only; state meta: at extraction

    def extract_result(self):
        if self.state['samples'] is None:
            raise ValueError('Nothing to extract')
        if self.adaptive and self.comm.on:
            with PHASES('extract:gather_adaptive'):
                self._gather_ranks_adaptive()
            self._update_state_meta()
        else:
            self._gather_ranks()
            self._update_state_meta()
            if self.adaptive:
                with PHASES('extract:update_distances'):
                    self._update_distances()
        n = self.objective['n_samples']
        # the arrays stay on the device; `outputs` copies a column to the host when it is read
        twins = {k: v[:n] for k, v in self.state['samples'].items()}
        sample = Sample(outputs=DeviceOutputs(twins), **self._extract_result_kwargs())
        sample._dev = twins
        if 'local_rows' in self.state:      # sharded summary columns of a multi-rank adaptive run
            sample.local_rows = self.state['local_rows']
            sample.local_summaries = self.state['local_summaries']
        return sample

    def _init_samples_lazy(self, batch):
        """Best-n buffers on the device (the reference keeps n + batch_size rows on the host,
        samplers.py:177-207; here the merge reads the batch in place)."""
        samples = {}
        n = self.objective['n_samples']
        for node in self.output_names:
            if node not in batch:
                raise KeyError("Did not receive outputs for node {}".format(node))
            nbatch = batch[node]
            if not em.is_array(nbatch):
                raise ValueError("Node {} output must be in a numpy array of length {} "
                                 "(batch_size).".format(node, self.batch_size))
            if len(nbatch) != self.batch_size:
                raise ValueError("Node {} output has array length {}. It should be equal to the "
                                 "batch size {}.".format(node, len(nbatch), self.batch_size))
            shape = (n,) + tuple(nbatch.shape[1:])
            if node == self.discrepancy_name:
                samples[node] = dev.full(shape, float('inf'))
            else:
                samples[node] = dev.zeros(shape)
        self.state['samples'] = samples

    def _merge_batch(self, batch):
        """samplers.py:209-237 on the device: accepted rows of the batch + current best-n ->
        sort by the (last) distance column -> gather the n smallest for every output."""
        samples = self.state['samples']
        n = self.objective['n_samples']
        dname = self.discrepancy_name
        if self.adaptive:
            self.model[dname].add_data(*[batch[s] for s in self.sums])

        d_batch = _to_dev_f64(batch[dname])
        acc = batch.get(('accepted', dname))
        if self.objective.get('threshold') is None and acc is None:
            map_b, n_cand = None, self.batch_size
        else:
            if acc is None:  # discrepancy node without fused acceptance (custom callable)
                thr = self.objective.get('threshold')
                if thr is None:
                    thr = self.state['threshold']
                ok = (d_batch <= dev.to_device(np.asarray(thr, dtype=np.float64)))
                if ok.dim() > 1:
                    ok = ok.all(dim=1)
                acc = torch.nonzero(ok).ravel().to(torch.int32)
            map_b, n_cand = acc, int(acc.numel())
        if self.objective.get('threshold') is not None:
            self._n_acceptable += n_cand
        if n_cand == 0:
            return
        # only the filled prefix of the best-n buffers takes part in the sort
        nv = self._n_valid
        n_out = min(n, nv + n_cand)
        key_state = samples[dname] if samples[dname].dim() == 1 else samples[dname][:, -1]
        key_batch = d_batch if d_batch.dim() == 1 else d_batch[:, -1]
        nodes = list(samples)
        tops = ops.merge_topn([samples[k][:nv] for k in nodes], [_to_dev_f64(batch[k]) for k in nodes],
                              key_state[:nv], key_batch, map_b, n_out)
        for node, top in zip(nodes, tops):
            if n_out == n:
                samples[node] = top
            else:
                samples[node][:n_out] = top
        self._n_valid = n_out

    def _update_state_meta(self):
        o, s = self.objective, self.state
        d = s['samples'][self.discrepancy_name]
        last = d[o['n_samples'] - 1]
        s['threshold'] = float(last.item()) if last.dim() == 0 else last.cpu().numpy()
        s['accept_rate'] = min(1, o['n_samples'] / s['n_sim'])

    def _update_objective_n_batches(self):
        """samplers.py:246-277.  n_acceptable = rows of the reference's (n + batch) buffer at or
        below the threshold = all rows accepted so far (the buffer never overflows before the
        sampler stops), tracked as a running count."""
        if self.objective.get('threshold') is None:
            return
        s = self.state
        n_samples = self.objective['n_samples']
        n_acceptable = self.comm.all_reduce_sum(self._n_acceptable) if self.comm.on \
            else self._n_acceptable
        n_sim = s['n_sim'] * self.comm.size if self.comm.on else s['n_sim']
        if n_acceptable == 0:
            n_batches = self.objective['n_batches'] + self._group
        else:
            accept_rate_t = n_acceptable / n_sim
            margin = .2 * self.batch_size * int(n_acceptable < n_samples)
            n_batches = ceil((n_samples / accept_rate_t + margin) / self.batch_size)
            if self.comm.on:
                n_batches = ceil(n_batches / self.comm.size)
        self.objective['n_batches'] = self._round_up_to_group(n_batches)

    def _update_distances(self):
        """samplers.py:279-299: append the new weight vector, re-score the kept rows with all
        K+1 nested distances, re-rank by the newest.  Like the reference, the distance output
        becomes the UNSORTED newest column while every other output is re-ordered."""
        node = self.model[self.discrepancy_name]
        node.update_distance()
        nums = self.objective['n_samples']
        data = {s: self.state['samples'][s][:nums] for s in self.sums}
        ds = node.generate(batch_size=nums, with_values=data)
        sort_distance = ds if ds.dim() == 1 else ds[:, -1].contiguous()
        sort_mask = ops.argsort(sort_distance)
        self.state['samples'][self.discrepancy_name] = sort_distance
        for k in self.state['samples'].keys():
            if k != self.discrepancy_name:
                self.state['samples'][k] = ops.take_rows(self.state['samples'][k], sort_mask)
        self._update_state_meta()

    def _gather_ranks(self):
        """Multi-GPU: ONE all-gather of the ranks' local best-n buffers -- every output packed into
        one (capacity, width) matrix -- then the same sort + gather on every rank, so all ranks
        hold the identical global best-n.  One small integer all-gather beforehand carries the
        per-rank row counts (-> common capacity) and the n_sim / n_batches totals."""
        if not self.comm.on or self._gathered:
            return
        self._gathered = True
        samples = self.state['samples']
        n = self.objective['n_samples']
        with PHASES('gather:counts'):
            counts = self.comm.all_gather_ints([self._n_valid, self.state['n_sim'],
                                                self.state['n_batches']])
        cap = max(1, min(n, ((int(counts[:, 0].max()) + 31) // 32) * 32))
        names = list(samples)
        shapes = {k: tuple(samples[k].shape[1:]) for k in names}
        widths = [int(np.prod(shapes[k])) if shapes[k] else 1 for k in names]
        offs = np.concatenate([[0], np.cumsum(widths)])
        with PHASES('gather:all_gather'):
            # rows beyond a rank's count carry +inf distances and sort last
            pack = torch.cat([samples[k][:cap].reshape(cap, w) for k, w in zip(names, widths)],
                             dim=1)
            allp = self.comm.all_gather_rows(pack)
        kcol = int(offs[names.index(self.discrepancy_name) + 1]) - 1      # last distance column
        with PHASES('gather:sort'):
            perm = ops.argsort(allp[:, kcol].contiguous())
        total = int(perm.numel())
        with PHASES('gather:select'):
            top = ops.take_rows(allp, perm[:min(n, total)])
            for k, w, o in zip(names, widths, offs[:-1]):
                col = top[:, o:o + w].reshape((top.shape[0],) + shapes[k])
                if total >= n:
                    samples[k] = col.contiguous()
                else:   # fewer than n rows exist globally: keep the padding of the local buffers
                    pad = samples[k][:n - total].clone()
                    pad.fill_(float('inf')) if k == self.discrepancy_name else pad.zero_()
                    samples[k] = torch.cat([col, pad])
        self._n_valid = min(n, int(counts[:, 0].sum()))
        self.state['n_sim'] = int(counts[:, 1].sum())
        self.state['n_batches'] = int(counts[:, 2].sum())
        if self.adaptive:
            self._merge_adaptive_moments()

    def _gather_ranks_adaptive(self):
        """Multi-GPU exchange of an adaptive-distance population WITHOUT moving the summaries
        (SURVEY.md section 8e, payload caveat).  The reference re-scores the kept rows centrally
        from their D summary columns (samplers.py:279-299); here
          1. the (n, mean, M2) column moments are Chan-merged (3 x D doubles per rank), so every
             rank derives the same new weight vector;
          2. each rank re-scores ITS OWN kept rows with all K + 1 nested distances;
          3. ONE all-gather moves [old ranking key | K + 1 new distances | parameters (+ outputs
             the caller asked for) | owner rank | local row] per kept row -- ~100 B instead of
             8 D + ... bytes;
          4. every rank selects the global best n by the old key and re-ranks them by the newest
             distance: the same rows, in the same order, as the central re-scoring.
        The summary columns of the selected rows stay on their owner ranks (`local_rows`: their
        positions in the population, `local_summaries`: the rows) unless asked for by name."""
        if self._gathered:
            return
        self._gathered = True
        samples = self.state['samples']
        n = self.objective['n_samples']
        dname = self.discrepancy_name
        node = self.model[dname]
        self._merge_adaptive_moments()
        node.update_distance()
        nv = self._n_valid
        counts = self.comm.all_gather_ints([nv, self.state['n_sim'], self.state['n_batches']])
        cap = max(1, min(n, ((int(counts[:, 0].max()) + 31) // 32) * 32))
        old = samples[dname]
        old_key = (old if old.dim() == 1 else old[:, -1])[:cap].reshape(cap, 1)
        k_new = len(node._s['w'])
        ds = dev.zeros((cap, k_new))
        if nv:
            ds[:nv] = node.generate(batch_size=nv, with_values={
                s: samples[s][:nv] for s in self.sums}).reshape(nv, k_new)
        sharded = [s for s in self.sums if s not in self._full_exchange]
        carried = [k for k in samples if k != dname and k not in sharded]
        shapes = {k: tuple(samples[k].shape[1:]) for k in carried}
        widths = [int(np.prod(shapes[k])) if shapes[k] else 1 for k in carried]
        owner = dev.full((cap, 1), float(self.comm.rank))
        local = dev.to_device(np.arange(cap, dtype=np.float64)).reshape(cap, 1)
        pack = torch.cat([old_key, ds] + [samples[k][:cap].reshape(cap, w)
                                          for k, w in zip(carried, widths)] + [owner, local], dim=1)
        allp = self.comm.all_gather_rows(pack)
        total = int(counts[:, 0].sum())
        m = min(n, total)
        top = ops.take_rows(allp, ops.argsort(allp[:, 0].contiguous())[:m])   # best n by the old key
        new_last = top[:, k_new].contiguous()
        order = ops.argsort(new_last)
        ranked = ops.take_rows(top, order)

        def padded(col, fill):
            if m == n:
                return col.contiguous()
            return torch.cat([col, dev.full((n - m,) + tuple(col.shape[1:]), fill)])
        # like the reference, the distance output is the UNSORTED newest column (samplers.py:294)
        samples[dname] = padded(new_last, float('inf'))
        off = 1 + k_new
        for k, w in zip(carried, widths):
            samples[k] = padded(ranked[:, off:off + w].reshape((m,) + shapes[k]), 0.0)
            off += w
        mine = torch.nonzero(ranked[:, off] == float(self.comm.rank)).reshape(-1)
        rows = ops.take_rows(ranked[:, off + 1].contiguous(), mine.to(torch.int32)).to(torch.int32)
        self.state['local_rows'] = mine
        self.state['local_summaries'] = {s: ops.take_rows(samples[s], rows) for s in sharded}
        for s in sharded:
            del samples[s]
        self._n_valid = m
        self.state['n_sim'] = int(counts[:, 1].sum())
        self.state['n_batches'] = int(counts[:, 2].sum())

    def _merge_adaptive_moments(self):
        """Chan-merge the per-rank (n, mean, M2) column moments (3 x D doubles per rank)."""
        st = self.model[self.discrepancy_name]._s
        n_r, m_r, s_r = st['store']
        D = np.size(m_r) if np.ndim(m_r) else 1
        pack = dev.zeros((1, 1 + 2 * D))
        pack[0, 0] = float(n_r)
        pack[0, 1:1 + D] = dev.to_device(np.broadcast_to(m_r, (D,)).copy())
        pack[0, 1 + D:] = dev.to_device(np.broadcast_to(s_r, (D,)).copy())
        allp = self.comm.all_gather_rows(pack).cpu().numpy()
        n0, m0, s0 = sharding.chan_merge([(row[0], row[1:1 + D], row[1 + D:]) for row in allp])
        st['store'] = [n0, m0, s0]
        st['scale'] = np.sqrt(s0 / n0)

    def iterate(self):
        """Batch index b is computed by rank b % world (each rank advances by world_size)."""
        if not self.comm.on:
            return super().iterate()
        batch_index = sharding.batch_index(self._next_batch_index, self.comm.rank, self.comm.size)
        values = self.prepare_new_batch(batch_index)
        self._next_batch_index += 1
        batch = self._run_batch(batch_index, values)
        self.update(batch, batch_index)


# ------------------------------------------------------------------------------------- SMC
class SMC(Sampler):
    """Sequential Monte Carlo ABC sampler (samplers.py:320-559)."""

    def __init__(self, model, discrepancy_name=None, output_names=None, device_proposal=None,
                 **kwargs):
        """`device_proposal` (optional, throughput mode): an object with
        ``rvs(means, cov, weights, size, key) -> (size, p) device tensor`` restricted to the prior
        support and ``logpdf(params) -> device tensor`` (e.g. examples.ma2.DeviceProposal); the
        default draws proposals from the host RandomState exactly like the reference."""
        model, discrepancy_name = self._resolve_model(model, discrepancy_name)
        if not hasattr(self, '_full_exchange'):
            self._full_exchange = set(n.name if isinstance(n, em.NodeReference) else n
                                      for n in (output_names or []))
        output_names = [discrepancy_name] + model.parameter_names + (output_names or [])
        super().__init__(model, output_names, **kwargs)
        self._prior = ModelPrior(self.model)
        self._device_proposal = device_proposal
        self.discrepancy_name = discrepancy_name
        self.state['round'] = 0
        self._populations = []
        self._rejection = None
        self._round_random_state = None
        self._quantiles = None
        self.bar = False

    def set_objective(self, n_samples, thresholds=None, quantiles=None):
        """One more population per entry of `thresholds` (or `quantiles`: the threshold of a
        round is then that quantile of the previous population's discrepancies), continuing
        after the populations already sampled."""
        schedule = thresholds if thresholds is not None else quantiles
        if schedule is None:
            raise ValueError('ABC-SMC needs either thresholds or quantiles')
        done = len(self._populations)
        self.state['round'] = done
        padded = np.concatenate((np.full(done, None), schedule))
        if thresholds is None:
            self._quantiles, thresholds = padded, np.full(len(padded), None)
        else:
            thresholds = padded
        self.objective.update(n_samples=n_samples, n_batches=self.max_parallel_batches,
                              round=len(padded) - 1, thresholds=thresholds)
        self._init_new_round()
        self._update_objective()

    def extract_result(self):
        pop = self._extract_population()
        self._populations.append(pop)
        return SmcSample(outputs=pop.outputs, populations=self._populations.copy(),
                         weights=pop.weights, threshold=pop.threshold,
                         **self._extract_result_kwargs())

    def _accept_hint(self):
        return self._rejection._accept_hint()

    def _extract_result_kwargs(self):
        kwargs = super()._extract_result_kwargs()
        if self.comm.on:      # the local counters cover this rank's batches only
            kwargs['n_sim'] = sum(pop.n_sim for pop in self._populations)
            kwargs['n_batches'] = sum(pop.n_batches for pop in self._populations)
        return kwargs

    def update(self, batch, batch_index):
        super().update(batch, batch_index)
        self._rejection.update(batch, batch_index)
        if self._rejection.finished:
            if self.state['round'] < self.objective['round']:
                self._populations.append(self._extract_population())
                self.state['round'] += 1
                self._init_new_round()
        self._update_objective()

    def iterate(self):
        if not self.comm.on:
            return super().iterate()
        batch_index = sharding.batch_index(self._next_batch_index, self.comm.rank, self.comm.size)
        with PHASES('prepare_new_batch'):
            values = self.prepare_new_batch(batch_index)
        self._next_batch_index += 1
        with PHASES('run_batch'):
            batch = self._run_batch(batch_index, values)
        with PHASES('update'):
            self.update(batch, batch_index)

    def prepare_new_batch(self, batch_index):
        if self.state['round'] == 0:
            return
        prev = self._populations[-1]
        if self._device_proposal is not None:
            # the proposal stream of a batch is a function of (round seed, global batch index)
            # only, so every sharding of the batches over ranks draws the same particles; the
            # component-draw table is built once per population
            if getattr(prev, '_cdf_dev', None) is None:
                prev._cdf_dev = ops.gm_cdf(None if prev._equal_weights else prev._w_dev,
                                           prev.n_samples)
            params = self._device_proposal.rvs(prev._means_dev, prev.cov, None, self.batch_size,
                                               _batch_key(self._round_seed, batch_index),
                                               cdf=prev._cdf_dev)
            return {p: params[:, i] for i, p in enumerate(self.parameter_names)}
        params = GMDistribution.rvs(prev.means, prev.cov, prev.weights, size=self.batch_size,
                                    prior_logpdf=self._prior.logpdf,
                                    random_state=self._round_random_state)
        params = params.reshape((-1, len(self.parameter_names)))
        return {p: params[:, i] for i, p in enumerate(self.parameter_names)}

    def _init_new_round(self):
        self._set_rejection_round(self.state['round'])
        if self.state['round'] == 0 and self._quantiles is not None:
            self._rejection.set_objective(self.objective['n_samples'], quantile=self._quantiles[0])
        else:
            if self._quantiles is not None:
                self._set_threshold()
            self._rejection.set_objective(self.objective['n_samples'],
                                          threshold=self.current_population_threshold)

    def _set_rejection_round(self, round):
        seed = self.seed if round == 0 else em.get_sub_seed(self.seed, round)
        self._round_seed = int(seed)
        host_seed = seed
        if self.comm.on and round > 0:
            # host proposals: each rank draws its own from the sequential host stream, so the
            # per-round streams are decorrelated by rank (device proposals are keyed per batch)
            host_seed = em.get_sub_seed(int(seed), self.comm.rank)
        self._round_random_state = np.random.RandomState(host_seed)
        self._rejection = Rejection(self.model, discrepancy_name=self.discrepancy_name,
                                    output_names=self.output_names, batch_size=self.batch_size,
                                    seed=seed, max_parallel_batches=self.max_parallel_batches,
                                    distributed=self._distributed)
        self._rejection._full_exchange = set(getattr(self, '_full_exchange', ()))
        self._population_cache = None

    def _extract_population(self):
        # extraction is a pure function of the finished rejection round; a second request (e.g.
        # AdaptiveThresholdSMC.extract_result after its update) gets the same object back
        if self._population_cache is not None and self._population_cache[0] is self._rejection:
            return self._population_cache[1]
        with PHASES('extract_result(gather)'):
            sample = self._rejection.extract_result()
        sample.method_name = "Rejection within SMC-ABC"
        with PHASES('weights_means_cov'):
            self._attach_weights_means_and_cov(sample)
        self._population_cache = (self._rejection, sample)
        return sample

    def _attach_weights_means_and_cov(self, sample):
        means, w, cov = self._compute_weights_means_and_cov(sample)
        sample.means = means
        sample.weights = w
        sample.meta['cov'] = cov

    def _compute_weights_means_and_cov(self, pop):
        """samplers.py:508-534 on the device: the O(N_new x N_prev) mixture density (sharded over
        the new particles when distributed, one all-gather of N doubles), the importance weights
        and the weighted variance.  Returns device arrays for means and weights (the sample
        object copies them to the host when they are read) and the host covariance matrix."""
        twins = pop._dev
        params_dev = torch.stack([twins[p].reshape(-1) for p in self.parameter_names], dim=1)
        N = int(params_dev.shape[0])
        if self._populations:
            prev = self._populations[-1]
            w_prev = None if prev._equal_weights else prev._w_dev
            if self.comm.on:
                lo, hi, per = sharding.shard_bounds(N, self.comm.rank, self.comm.size)
                q_part = dev.full((per,), float('nan'))
                with PHASES('weights:gm_logpdf'):
                    if hi > lo:
                        q_part[:hi - lo] = ops.gm_logpdf(params_dev[lo:hi], prev._means_dev,
                                                         prev.cov, w_prev, validate=False,
                                                         mixed=self._device_proposal is not None)
                with PHASES('weights:all_gather'):
                    q_logpdf = self.comm.all_gather_rows(q_part)
                q_logpdf = q_logpdf[:N]   # equal-capacity shards: only the tail is padding
            else:
                with PHASES('weights:gm_logpdf'):
                    q_logpdf = ops.gm_logpdf(params_dev, prev._means_dev, prev.cov, w_prev,
                                             validate=False,
                                             mixed=self._device_proposal is not None)
            with PHASES('weights:prior_logpdf'):
                if self._device_proposal is not None:
                    p_logpdf = self._device_proposal.logpdf(params_dev)
                else:
                    p_logpdf = self._prior.logpdf(dev.to_host(params_dev))
            w_dev = ops.smc_weights(p_logpdf, q_logpdf)
            if not bool((w_dev != 0).any()):
                raise RuntimeError("All sample weights are zero. If you are using a prior "
                                   "with a bounded support, this may be caused by specifying "
                                   "a too small sample size.")
        else:
            w_dev = None
        pop._means_dev = params_dev
        pop._equal_weights = w_dev is None
        pop._w_dev = w_dev
        with PHASES('weights:weighted_var'):
            cov = 2 * np.diag(ops.weighted_var(params_dev, w_dev))
        if not np.all(np.isfinite(cov)):
            logger.warning("Could not estimate the sample covariance. This is often "
                           "caused by majority of the sample weights becoming zero."
                           "Falling back to using unit covariance.")
            cov = np.diag(np.ones(params_dev.shape[1]))
        return params_dev, (w_dev if w_dev is not None else np.ones(N)), cov

    def _update_objective(self):
        n_batches = sum([pop.n_batches for pop in self._populations])
        if self.comm.on:
            n_batches = ceil(n_batches / self.comm.size)
        self.objective['n_batches'] = n_batches + self._rejection.objective['n_batches']

    def _set_threshold(self):
        prev = self._populations[self.state['round'] - 1]
        d_prev = prev._dev[self.discrepancy_name]
        # equal weights (round 0) have the same arithmetic as weights=None: closed form
        w_prev = None if prev._equal_weights else prev._w_dev
        with PHASES('weighted_quantile'):
            threshold = ops.weighted_sample_quantile(d_prev, self._quantiles[self.state['round']],
                                                     w_prev)
        self.objective['thresholds'][self.state['round']] = threshold

    @property
    def current_population_threshold(self):
        return self.objective['thresholds'][self.state['round']]


class AdaptiveDistanceSMC(SMC):
    """SMC-ABC with adaptive threshold and distance (Prangle 2017 Alg. 5); samplers.py:562-659."""

    def __init__(self, model, discrepancy_name=None, output_names=None, **kwargs):
        model, discrepancy_name = self._resolve_model(model, discrepancy_name)
        if not isinstance(model[discrepancy_name], em.AdaptiveDistance):
            raise TypeError('This method requires an adaptive distance node.')
        model[discrepancy_name].init_state()
        sums = [s.name for s in model[discrepancy_name].parents]
        self._full_exchange = set(n.name if isinstance(n, em.NodeReference) else n
                                  for n in (output_names or []))
        if output_names is None:
            output_names = sums
        else:
            for k in sums:
                if k not in output_names:
                    output_names.append(k)
        super().__init__(model, discrepancy_name, output_names=output_names, **kwargs)

    def set_objective(self, n_samples, rounds, quantile=0.5):
        super().set_objective(ceil(n_samples / quantile), quantiles=[1] * rounds)
        self.population_size = n_samples
        self.quantile = quantile

    def _extract_population(self):
        if self._population_cache is not None and self._population_cache[0] is self._rejection:
            return self._population_cache[1]
        rejection_sample = self._rejection.extract_result()
        ps = self.population_size
        twins = {k: rejection_sample._dev[k][:ps] for k in self.output_names
                 if k in rejection_sample._dev}
        meta = rejection_sample.meta
        meta['adaptive_distance_w'] = self.model[self.discrepancy_name]._s['w'][-1]
        meta['threshold'] = float(twins[self.discrepancy_name].max().item())
        meta['accept_rate'] = self.population_size / meta['n_sim']
        sample = Sample("Rejection within adaptive distance SMC-ABC", DeviceOutputs(twins),
                        self.parameter_names, **{k: v for k, v in meta.items()
                                                 if k not in ('method_name', 'parameter_names')})
        sample._dev = twins
        rows = getattr(rejection_sample, 'local_rows', None)
        if rows is not None:    # multi-rank: this rank's share of the population's summaries
            keep = rows < ps
            sample.local_rows = rows[keep]
            sample.local_summaries = {s: v[keep] for s, v in
                                      rejection_sample.local_summaries.items()}
        self._attach_weights_means_and_cov(sample)
        self._population_cache = (self._rejection, sample)
        return sample

    def _extract_result_kwargs(self):
        kwargs = super()._extract_result_kwargs()
        kwargs['adaptive_distance_w'] = [pop.adaptive_distance_w for pop in self._populations]
        return kwargs

    def _set_threshold(self):
        round = self.state['round']
        self.objective['thresholds'][round] = self._populations[round - 1].threshold

    @property
    def current_population_threshold(self):
        return [np.inf] + [pop.threshold for pop in self._populations]


# --------------------------------------------------------------------- adaptive threshold SMC
def calculate_densratio_basis_sigma(sigma_1, sigma_2):
    """elfi/methods/density_ratio_estimation.py:11-31."""
    return sigma_1 * sigma_2 / np.sqrt(np.abs(sigma_1 ** 2 - sigma_2 ** 2))


class DensityRatioEstimation:
    """KLIEP density-ratio estimation on the device (density_ratio_estimation.py:34-207).
    Only the fixed-sigma path (optimize=False) that AdaptiveThresholdSMC uses is implemented."""

    def __init__(self, n=100, epsilon=0.1, max_iter=500, abs_tol=0.01, conv_check_interval=20,
                 fold=5, optimize=False):
        if optimize:
            raise NotImplementedError('likelihood cross-validation of the RBF scale is not '
                                      'implemented on the device')
        self.n = n
        self.epsilon = epsilon
        self.max_iter = max_iter
        self.abs_tol = abs_tol
        self.fold = fold
        self.sigma = None
        self.conv_check_interval = conv_check_interval
        self.optimize = False
        self._max_ratio = None
        self.alpha = None

    def fit(self, x, y, weights_x=None, weights_y=None, sigma=None):
        if isinstance(sigma, (float, np.floating)):
            self.sigma = float(sigma)
        if self.sigma is None:
            raise ValueError("RBF width (sigma) has to provided in first call.")
        x, y = [v if dev.is_device_array(v) else np.asarray(v, dtype=np.float64) for v in (x, y)]
        x = x.reshape(x.shape[0], -1)
        y = y.reshape(y.shape[0], -1)
        self.alpha, self._max_ratio, self.n_iter = ops.kliep_fit(
            x, y, weights_x, weights_y, sigma=self.sigma, n_basis=self.n, epsilon=self.epsilon,
            max_iter=self.max_iter, abs_tol=self.abs_tol,
            conv_check_interval=self.conv_check_interval)

    def max_ratio(self):
        return self._max_ratio


class AdaptiveThresholdSMC(SMC):
    """ABC-SMC with adaptive threshold selection (Simola et al. 2021); samplers.py:662-840."""

    def __init__(self, model, discrepancy_name=None, output_names=None, initial_quantile=0.20,
                 q_threshold=0.99, densratio_estimation=None, **kwargs):
        super().__init__(model, discrepancy_name, output_names, **kwargs)
        # Multi-rank: after the gather every rank holds the same population, the KLIEP fit is
        # deterministic, and the prior reference sample of the first fit comes from the round-0
        # RandomState, which is seeded identically on all ranks and not used for proposals -- so
        # every rank derives the same quantile without a collective.
        self.q_threshold = q_threshold
        self.initial_quantile = initial_quantile
        self.densratio = densratio_estimation or DensityRatioEstimation(
            n=100, epsilon=0.001, max_iter=200, abs_tol=0.01, fold=5, optimize=False)

    def set_objective(self, n_samples, max_iter=10):
        rounds = max_iter - 1
        self.state['round'] = len(self._populations)
        rounds = rounds + self.state['round']
        thresholds = np.full((rounds + 1), None)
        self._quantiles = np.full((rounds + 1), None)
        self._quantiles[0] = self.initial_quantile
        self.objective.update(dict(n_samples=n_samples, n_batches=self.max_parallel_batches,
                                   round=rounds, thresholds=thresholds))
        self._init_new_round()
        self._update_objective()

    def update(self, batch, batch_index):
        ParameterInference.update(self, batch, batch_index)
        self._rejection.update(batch, batch_index)
        if self._rejection.finished:
            self._new_population = self._extract_population()
            if self.state['round'] < self.objective['round']:
                self._set_adaptive_quantile()
                if self._quantiles[self.state['round'] + 1] < self.q_threshold:
                    self._populations.append(self._new_population)
                    self.state['round'] += 1
                    self._init_new_round()
        self._update_objective()

    def extract_result(self):
        # the reference extracts the last population again through SMC.extract_result; here the
        # population of the finished round is extracted (and, multi-rank, gathered) exactly once
        return super().extract_result()

    def _set_adaptive_quantile(self):
        cur = self._resolve_sample(backwards_index=0)
        prev = self._resolve_sample(backwards_index=-1)
        sigma = calculate_densratio_basis_sigma(cur['sigma_max'], prev['sigma_max'])
        self.densratio.fit(x=cur['samples'], y=prev['samples'], weights_x=cur['weights'],
                           weights_y=prev['weights'], sigma=float(sigma))
        max_value = self.densratio.max_ratio()
        max_value = 1.0 if max_value < 1.0 else max_value
        self._quantiles[self.state['round'] + 1] = max(1 / max_value, 0.05)

    def _resolve_sample(self, backwards_index):
        if self.state['round'] + backwards_index < 0:
            return self._densityratio_initial_sample()
        sample = self._new_population if backwards_index == 0 else self._populations[backwards_index]
        sample_sigma = np.sqrt(np.diag(sample.cov))
        return dict(samples=sample._means_dev,
                    weights=None if sample._equal_weights else sample._w_dev,
                    sigma_max=np.min(sample_sigma))

    def _densityratio_initial_sample(self):
        n_samples = self._new_population.weights.shape[0]
        samples = self._prior.rvs(size=n_samples, random_state=self._round_random_state)
        weights = np.ones(n_samples)
        sample_cov = np.atleast_2d(np.cov(samples.reshape(n_samples, -1), rowvar=False))
        return dict(samples=samples, weights=weights,
                    sigma_max=np.min(np.sqrt(np.diag(sample_cov))))
