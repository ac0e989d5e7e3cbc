"""Testbench: compare inference methods over repeated observations (elfi/testbench/testbench.py).

A Testbench infers one model `repetitions` times with each added method, once per observation
simulated from the reference parameters, and reports per-parameter sample-mean errors.  Names,
arguments, result layouts and the seeding order are the reference's, quirks included (DESIGN.md
section 7, "Testbench").

`run()` steps the R repetitions of two kinds of method together (lock-step); every other method
runs its repetitions one after the other.  Each repetition keeps its own model copy, observation,
seed and plan, and its result is bit-identical to its serial run, method(model_r, seed=seed_r)
.sample(...).

* Rejection in quantile or n_sim mode consumes the same number of batches in every repetition.
  Per batch index, the summaries of all R go into one (R B, D) device matrix, one segmented
  distance launch (ops.dist_seg) measures every block against its own observation, and one
  segmented top-n merge (ops.merge_topn_seg) updates all R best-n buffers.
* BSL with a device likelihood (any n_chains, with or without device_proposal).  Per iteration
  every unfinished repetition simulates its own round into its block of one (R C, n_sim_round, d)
  device feature buffer, one ops.synlik call evaluates the R C groups against their own
  observations, and one device-to-host read of R C values feeds each repetition's host
  Metropolis-Hastings step.  Repetitions whose proposals all leave the prior support skip rounds,
  so they progress raggedly; a finished repetition's group is evaluated and ignored.  In
  throughput mode (device_proposal) the chains of all repetitions live in stacked device buffers
  and one keyed ops.bsl_mh_step steps them all, each with its own seed as Philox key: no read
  happens between the first round's check and the end.
"""
import functools
import logging
import sys

import numpy as np
import torch

from . import bsl
from . import device as dev
from . import model as em
from . import ops
from .samplers import Comm, Rejection, _to_dev_f64
from .throughput import LazySimulation

logger = logging.getLogger(__name__)

__all__ = ['Testbench', 'TestbenchMethod']


class _ProgressBar:
    """Text progress bar of the reference (elfi/visualization/visualization.py ProgressBar)."""

    def __init__(self, prefix='', suffix='', decimals=1, length=100, fill='='):
        self.prefix, self.suffix = prefix, suffix
        self.decimals, self.length, self.fill = decimals, length, fill
        self.finished = False

    def update_progressbar(self, iteration, total):
        if self.finished:
            return
        percent = ('{0:.' + str(self.decimals) + 'f}').format(100 * (iteration / float(total)))
        filled = int(self.length * iteration // total)
        bar = self.fill * filled + '-' * (self.length - filled)
        sys.stdout.write('\r%s [%s] %s%% %s' % (self.prefix, bar, percent, self.suffix))
        if iteration == total:
            sys.stdout.write('\n')
            self.finished = True
        sys.stdout.flush()

    def reinit_progressbar(self, scaling=0, reinit_msg=None):
        self.finished = False
        if reinit_msg:
            sys.stdout.write('\n' + reinit_msg + '\n')


def _to_host(x):
    """Simulator or prior output as host data (device models return device arrays or lazy
    simulator output; observations are host data)."""
    if isinstance(x, LazySimulation):
        x = x.materialize()
    return dev.to_host(x) if dev.is_device_array(x) else x


class Testbench:
    """Base class for comparing the performance of LFI-methods.

    One model is inferred `repetitions` times with each of the methods added by `add_method`.
    """

    def __init__(self, model=None, repetitions=1, observations=None, reference_parameter=None,
                 reference_posterior=None, progress_bar=True, seed=None):
        self.model = model
        self.method_list = []
        self.method_seed_list = []
        self.repetitions = repetitions
        self.rng = np.random.RandomState(seed)

        self.observations = observations.copy() if observations is not None else observations
        self.reference_parameter = reference_parameter.copy() \
            if reference_parameter is not None else reference_parameter

        self.param_dim = len(model.parameter_names)
        self.param_names = model.parameter_names
        self.reference_posterior = reference_posterior
        self.simulator_name = list(model.observed)[0]
        if progress_bar:
            self.progress_bar = _ProgressBar(prefix='Progress', suffix='Complete', decimals=1,
                                             length=50, fill='=')
        else:
            self.progress_bar = None

        self._resolve_test_type()
        self._collect_tests()

    def _collect_tests(self):
        self.test_dictionary = {
            'model': self.model,
            'observations': self.observations,
            'reference_parameter': self.reference_parameter,
            'reference_posterior': self.reference_posterior
        }

    def _get_seeds(self, n_rep=1):
        """Fix a seed for each of the repeated instances."""
        return self.rng.randint(low=0, high=2 ** 32 - 1, size=n_rep, dtype=np.uint32)

    def _resolve_test_type(self):
        self._set_default_test_type()
        self._resolve_observations()
        self._resolve_reference_parameters()

    def _set_default_test_type(self):
        self.description = {
            'observations_available': self.observations is not None,
            'reference_parameters_available': self.reference_parameter is not None,
            'reference_posterior_available': self.reference_posterior is not None
        }

    def _resolve_reference_parameters(self):
        if self.description['reference_parameters_available']:
            for keys, values in self.reference_parameter.items():
                self.reference_parameter[keys] = np.repeat(_to_host(values),
                                                           repeats=self.repetitions)
        elif not self.description['observations_available']:
            seed = self._get_seeds(n_rep=1)
            params = self.model.generate(batch_size=self.repetitions,
                                         outputs=self.model.parameter_names, seed=seed[0])
            self.reference_parameter = {k: _to_host(v) for k, v in params.items()}

    def _resolve_observations(self):
        if self.description['observations_available']:
            self.observations = np.repeat(self.observations, repeats=self.repetitions, axis=0)
        else:
            seed = self._get_seeds(n_rep=1)
            self.observations = _to_host(self.model.generate(
                with_values=self.reference_parameter, outputs=self.simulator_name,
                batch_size=self.repetitions, seed=seed[0])[self.simulator_name])

    def add_method(self, new_method):
        """Add a new method (a TestbenchMethod) to the testbench."""
        logger.info('Adding {} to testbench.'.format(new_method.attributes['name']))
        self.method_list.append(new_method)
        self.method_seed_list.append(self._get_seeds(n_rep=self.repetitions))

    def run(self, lockstep=True):
        """Run Testbench.  With `lockstep`, a Rejection method in quantile or n_sim mode and a BSL
        method with a device likelihood run their repetitions together (see the module
        docstring); every other method, and every method with ``lockstep=False``, runs its
        repetitions one after the other."""
        self.testbench_results = []
        for method_index, method in enumerate(self.method_list):
            logger.info('Running {} in testbench.'.format(method.attributes['name']))

            if self.progress_bar:
                self.progress_bar.reinit_progressbar(reinit_msg=method.attributes['name'])

            seeds = self.method_seed_list[method_index]
            metric = self._lockstep_metric(method) if lockstep else None
            if metric is not None:
                result = self._collect_results(method.attributes['name'],
                                               self._lockstep_rejection(method, seeds, *metric))
            elif lockstep and self._lockstep_bsl_applies(method):
                result = self._collect_results(method.attributes['name'],
                                               self._lockstep_bsl(method, seeds))
            else:
                result = self._repeat_inference(method, seeds)
            self.testbench_results.append(result)

    def _repeat_inference(self, method, seed_list):
        repeated_result = []
        model = self.model.copy()
        for i in np.arange(self.repetitions):
            if self.progress_bar:
                self.progress_bar.update_progressbar(i + 1, self.repetitions)

            model.observed[self.simulator_name] = np.atleast_2d(self.observations[i])

            repeated_result.append(self._draw_posterior_sample(method, model, seed_list[i]))

        return self._collect_results(method.attributes['name'], repeated_result)

    def _draw_posterior_sample(self, method, model, seed):
        method_instance = method.attributes['callable'](
            model, **method.attributes['method_kwargs'], seed=seed)

        fit_kwargs = method.attributes['fit_kwargs']

        if len(fit_kwargs) > 0:
            method_instance.fit(fit_kwargs)

        sampler_kwargs = method.attributes['sample_kwargs']

        return method_instance.sample(**sampler_kwargs)

    def _collect_results(self, name, results):
        return {'method': name, 'results': results}

    def _compare_sample_results(self):
        """Compare results in sample-format."""

    def _retrodiction(self):
        """Infer a problem with known parameter values."""

    def get_testbench_results(self):
        """Return Testbench testcases and results."""
        return {'testcases': self.test_dictionary, 'results': self.testbench_results}

    def parameterwise_sample_mean_differences(self):
        """Return parameterwise differences for the sample mean for methods in Testbench."""
        sample_mean_difference_results = {}
        for method_results in self.testbench_results:
            sample_mean_difference_results[method_results['method']] = (
                self._get_sample_mean_difference(method_results))
        return sample_mean_difference_results

    def _get_sample_mean_difference(self, method):
        sample_mean_difference = {}
        for param_names in self.param_names:
            sample_mean_difference[param_names] = [
                results.sample_means[param_names] - self.reference_parameter[param_names][0]
                for results in method['results']
            ]
        return sample_mean_difference

    # -- lock-step Rejection -----------------------------------------------------------------
    def _lockstep_metric(self, method):
        """(metric, p) of the segmented distance when `method` runs in lock-step, else None:
        this package's Rejection without fit kwargs, a pool or a threshold, on one rank, with a
        plain Distance whose metric ops.dist_seg computes."""
        a = method.attributes
        mk, sk = a['method_kwargs'], a['sample_kwargs']
        if a['callable'] is not Rejection or a['fit_kwargs'] or mk.get('pool') is not None:
            return None
        if sk.get('threshold') is not None or Comm(mk.get('distributed', True)).on:
            return None
        dname = mk.get('discrepancy_name')
        dname = dname.name if isinstance(dname, em.NodeReference) else dname
        if not isinstance(dname, str) or not self.model.has_node(dname):
            return None
        rec = self.model.record(dname)
        op = rec.op
        if rec.cls is not em.Distance or not isinstance(op, functools.partial):
            return None
        if op.func is em.device_euclidean_discrepancy and op.keywords.get('w') is None:
            return 'euclidean', 2.0
        if op.func is em.device_metric_discrepancy:
            return op.args[0], op.keywords.get('p', 2.0)
        return None

    def _lockstep_rejection(self, method, seed_list, metric, p):
        a = method.attributes
        skw = {k: v for k, v in a['sample_kwargs'].items() if k not in ('bar', 'vis')}
        R = self.repetitions
        model = self.model.copy()
        reps = []
        for i in range(R):
            model.observed[self.simulator_name] = np.atleast_2d(self.observations[i])
            reps.append(Rejection(model, **a['method_kwargs'], seed=seed_list[i]))
        for rej in reps:
            rej.set_objective(**skw)
        first = reps[0]
        dname = first.discrepancy_name
        parents = first.model.get_parents(dname)
        twin = em.observed_name(dname)
        wanted = list(dict.fromkeys([k for k in first.output_names if k != dname] + parents))
        plans = [em.compile_plan(rej.model, wanted + [twin]) for rej in reps]
        n = first.objective['n_samples']
        B = first.batch_size
        n_batches = first.objective['n_batches']
        S_all = obs_all = big = nodes = None
        nv = 0
        for b in range(n_batches):
            if self.progress_bar:
                self.progress_bar.update_progressbar(b + 1, n_batches)
            batches = []
            for r, (rej, plan) in enumerate(zip(reps, plans)):
                batch = em.execute_batch(rej.model, wanted + [twin], rej.computation_context, b,
                                         compiled=plan)
                rej.computation_context.num_submissions += 1
                rej.state['n_batches'] += 1
                rej.state['n_sim'] += B
                X = em._stack_summaries([batch[s] for s in parents])
                if S_all is None:
                    S_all = dev.empty((R * B, X.shape[1]))
                S_all[r * B:(r + 1) * B] = X
                batches.append(batch)
            if obs_all is None:
                rows = [em._stack_observed(batch[twin]) for batch in batches]
                if any(row.shape[0] != 1 for row in rows):
                    raise ValueError('observed summaries must form a single row')
                obs_all = dev.to_device(np.concatenate(rows))
            d_all = ops.dist_seg(S_all, obs_all, metric, p)
            key_batch = d_all.reshape(R, B)
            if big is None:
                for r, (rej, batch) in enumerate(zip(reps, batches)):
                    rej._init_samples_lazy(dict(batch, **{dname: key_batch[r]}))
                nodes = list(first.state['samples'])
                big = {k: torch.stack([rej.state['samples'][k] for rej in reps]) for k in nodes}
            new = [key_batch if k == dname else
                   torch.stack([_to_dev_f64(batch[k]) for batch in batches]) for k in nodes]
            n_out = min(n, nv + B)
            tops = ops.merge_topn_seg([big[k][:, :nv] for k in nodes], new, big[dname][:, :nv],
                                      key_batch, n_out)
            for k, top in zip(nodes, tops):
                if n_out == n:
                    big[k] = top
                else:
                    big[k][:, :n_out] = top
            nv = n_out
        results = []
        for r, rej in enumerate(reps):
            rej.state['samples'] = {k: big[k][r] for k in nodes}
            rej._n_valid = nv
            results.append(rej.extract_result())
        return results

    # -- lock-step BSL -----------------------------------------------------------------------
    @staticmethod
    def _lockstep_bsl_applies(method):
        """Whether `method` is this package's BSL, without fit kwargs or a pool, with a device
        likelihood (standard or unbiased)."""
        a = method.attributes
        mk = a['method_kwargs']
        return (a['callable'] is bsl.BSL and not a['fit_kwargs'] and mk.get('pool') is None
                and bsl._device_likelihood(mk.get('likelihood')) is not None)

    def _lockstep_bsl(self, method, seed_list):
        a = method.attributes
        sk = a['sample_kwargs']
        R = self.repetitions
        model = self.model.copy()
        reps = []
        for i in range(R):
            model.observed[self.simulator_name] = np.atleast_2d(self.observations[i])
            reps.append(bsl.BSL(model, **a['method_kwargs'], seed=seed_list[i]))
        first = reps[0]
        n_samples = int(sk['n_samples'])
        C = int(sk.get('n_chains', 1))
        d, b = first.observed.size, first._rows_per_chain
        state = None
        if first.device_proposal is not None:
            p = len(sk.get('param_names') or first.model.parameter_names)
            state = dict(chains=dev.zeros((R * C, n_samples, p)),
                         logpost=dev.zeros((R * C, n_samples)),
                         n_acc=dev.zeros((R * C,), dtype=torch.int64),
                         prop=dev.zeros((R * C, p)), prop_lp=dev.zeros((R * C,)),
                         rows=dev.zeros((p, R * C * b)))
        feats = dev.zeros((R * C, first.n_sim_round, d))
        for r, rep in enumerate(reps):
            block = slice(r * C, (r + 1) * C)
            rep._set_up(**sk, device_state=None if state is None else dict(
                {k: v[block] for k, v in state.items() if k != 'rows'},
                rows=state['rows'][:, r * C * b:(r + 1) * C * b]))
            rep.set_objective(n_samples)
            rep._sim = feats[block] if C > 1 else feats[r * C]
        obs = dev.to_device(np.repeat(np.concatenate([rep.observed.reshape(1, d) for rep in reps]),
                                      C, axis=0))
        lik = first._device_lik
        if state is not None:
            keys = dev.to_device(np.repeat(np.asarray(seed_list[:R], dtype=np.int64), C),
                                 dtype=torch.int64)
            lanes = dev.to_device(np.tile(np.arange(C, dtype=np.int32), R), dtype=torch.int32)
        while True:
            live = [rep for rep in reps if not rep.finished]
            if not live:
                break
            if self.progress_bar:
                self.progress_bar.update_progressbar(
                    max(rep.state['n_samples'] for rep in live) + 1, n_samples)
            for rep in live:
                rep._simulate_round()
            ll = lik.device(feats, obs)
            if state is None:
                ll = dev.to_host(ll)          # the one device-to-host read of the iteration
                for r, rep in enumerate(reps):
                    if rep in live:
                        rep._step(ll[r * C:(r + 1) * C])
            else:
                t = first.state['n_samples']          # every repetition runs every round
                if t == 0:
                    host = dev.to_host(ll)            # the one read of throughput mode
                    for r, rep in enumerate(reps):
                        rep._check_first_round(host[r * C:(r + 1) * C])
                ops.bsl_mh_step(first._tables, t, ll, state['prop'], state['prop_lp'],
                                state['chains'], state['logpost'], state['n_acc'], state['rows'],
                                keys, first.burn_in, lanes=lanes)
                for rep in live:
                    rep.state['n_samples'] += 1
            for rep in live:
                rep._end_round()
        return [rep.extract_result() for rep in reps]


class TestbenchMethod:
    """Container for ParameterInference methods included in Testbench."""

    def __init__(self, method, method_kwargs={}, fit_kwargs={}, sample_kwargs={}, name=None):
        name = name or method.__name__
        self.attributes = {'callable': method,
                           'method_kwargs': method_kwargs,
                           'fit_kwargs': fit_kwargs,
                           'sample_kwargs': sample_kwargs,
                           'name': name}

    def set_method_kwargs(self, **kwargs):
        """Add options for the ParameterInference contructor."""
        logger.info("Setting options for {}".format(self.attributes['name']))
        self.attributes['method_kwargs'] = kwargs

    def set_fit_kwargs(self, **kwargs):
        """Add options for the ParameterInference method fit()."""
        logger.info("Setting surrogate fit options for {}".format(self.attributes['name']))
        self.attributes['fit_kwargs'] = kwargs

    def set_sample_kwargs(self, **kwargs):
        """Add options for the ParameterInference method sample()."""
        logger.info("Setting sampler options for {}".format(self.attributes['name']))
        self.attributes['sample_kwargs'] = kwargs

    def get_method(self):
        """Return TestbenchMethod attributes."""
        return self.attributes
