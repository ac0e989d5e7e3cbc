"""Summary-statistic selection: the two-stage procedure of Nunes and Balding (2010)
(elfi/methods/diagnostics.py).

Every candidate combination of summaries is scored by the entropy of the parameters its rejection
sample accepts (stage 1), and by the mean root sum of squared errors of those parameters around
the parameters of the datasets closest to the data under the minimum-entropy combination
(stage 2).

For the cdist metrics 'euclidean', 'sqeuclidean', 'cityblock' and 'chebyshev' the batches are
simulated once and kept on the device with every candidate summary: one kernel scores all
combinations per row, and each combination keeps its best rows in the order
``Rejection(..., batch_size, seed).sample(n_acc, n_sim=n_sim)`` returns them.  Other metrics and
callables run the reference's loop, one rejection sampler per combination.  Both paths score the
accepted parameters with the same kernels (ops.knn_entropy, ops.mrsse).
"""
import logging
from itertools import combinations
from math import ceil

import numpy as np
import torch
from scipy.special import digamma, gamma

from . import device as dev
from . import model as em
from . import ops
from .samplers import Comm, Rejection
from .store import OutputPool

logger = logging.getLogger(__name__)

# metrics whose all-combination kernel is bit-identical to cdist (ops.subset_distance)
DEVICE_METRICS = tuple(ops.SUBSET_METRIC_CODES)
# the (combinations x rows) block of distances computed at a time stays within this
DISTANCE_BLOCK_BYTES = 256 << 20


class TwoStageSelection:
    """Perform the summary-statistics selection proposed by Nunes and Balding (2010).

    The user can provide a list of summary statistics as list_ss, and let the class combine them
    (every combination up to ``max_cardinality`` candidates, cardinality 1 first), or provide
    already combined summary statistics as prepared_ss (lists of callables are accepted as well
    as tuples).  After :meth:`run`, ``scores`` holds one record per combination: its ``names``,
    ``entropy`` and ``mrsse``.

    References
    ----------
    [1] Nunes, M. A., & Balding, D. J. (2010).
    On optimal selection of summary statistics for approximate Bayesian computation.
    Statistical applications in genetics and molecular biology, 9(1).
    [2] Blum, M. G., Nunes, M. A., Prangle, D., & Sisson, S. A. (2013).
    A comparative review of dimension reduction methods in approximate Bayesian computation.
    Statistical Science, 28(2), 189-208.
    """

    def __init__(self, simulator, fn_distance, list_ss=None, prepared_ss=None,
                 max_cardinality=4, seed=0):
        """`simulator` is the node the summaries apply to; `fn_distance` a cdist metric name or
        a callable discrepancy, as for Distance / Discrepancy."""
        if list_ss is None and prepared_ss is None:
            raise ValueError('No summary statistics to assess.')
        self.simulator = simulator
        self.fn_distance = fn_distance
        self.seed = seed
        if prepared_ss is not None:
            self.ss_candidates = [tuple(set_ss) for set_ss in prepared_ss]
        else:
            self.ss_candidates = self._combine_ss(list_ss, max_cardinality=max_cardinality)
        # the rejection runs of the per-combination loop share the simulator's outputs
        self.pool = OutputPool([simulator.name])
        self.scores = None

    def _combine_ss(self, list_ss, max_cardinality):
        """All combinations of list_ss of up to max_cardinality candidates, in
        itertools.combinations order, cardinality 1 first."""
        if max_cardinality > len(list_ss):
            max_cardinality = len(list_ss)
        combinations_ss = []
        for i in range(max_cardinality):
            for combination in combinations(list_ss, i + 1):
                combinations_ss.append(combination)
        return combinations_ss

    def run(self, n_sim, n_acc=None, n_closest=None, batch_size=1, k=4):
        """Run the two-stage procedure and return the combination with the minimum MRSSE.

        `n_acc` defaults to int(n_sim / 100) and `n_closest` to int(n_acc / 100); `k` is the
        neighbour of the entropy estimate (1 <= k <= 32).  Accepted parameters have at most 16
        dimensions."""
        if n_acc is None:
            n_acc = int(n_sim / 100)
        if n_closest is None:
            n_closest = int(n_acc / 100)
        if n_sim < n_acc or n_acc < n_closest or n_closest == 0:
            raise ValueError("The number of simulations is too small.")
        if Comm().on:
            raise RuntimeError('TwoStageSelection runs on one rank; it was called in a '
                               'torch.distributed group of several ranks')
        if isinstance(self.fn_distance, str) and self.fn_distance in DEVICE_METRICS:
            thetas = self._device_accepted_thetas(n_sim, n_acc, batch_size)
        else:
            thetas = torch.stack([self._obtain_accepted_thetas(set_ss, n_sim, n_acc, batch_size)
                                  for set_ss in self.ss_candidates])
        return self._select(thetas, n_acc, n_closest, k)

    # ---- stage 1 and 2 on the accepted parameters (C, n_acc, q) ---------------------------------
    @staticmethod
    def _entropy(q, n_acc, k, sum_log_dist_knn):
        """diagnostics.py:249-252, with the sum of the log radii from the device."""
        return np.log(np.pi**(q / 2) / gamma((q / 2) + 1)) - digamma(k) \
            + np.log(n_acc) + (q / n_acc) * sum_log_dist_knn

    def _select(self, thetas, n_acc, n_closest, k):
        q = int(thetas.shape[2])
        _, logsum = ops.knn_entropy(thetas, k)
        entropies = [self._entropy(q, n_acc, k, s) for s in dev.to_host(logsum)]
        names = [[ss.__name__ for ss in set_ss] for set_ss in self.ss_candidates]

        E_me = np.inf
        names_ss_me = []
        i_me = None
        for i, (names_ss, E_ss) in enumerate(zip(names, entropies)):
            # If equal, dismiss the combination which contains uninformative summary statistics.
            if (E_ss == E_me and (len(names_ss_me) > len(names_ss))) or E_ss < E_me:
                E_me = E_ss
                names_ss_me = names_ss
                i_me = i
            logger.info('Combination %s shows the entropy of %f' % (names_ss, E_ss))
        # Note: entropy is in the log space (negative values allowed).
        logger.info('\nThe minimum entropy of %f was found in %s.\n' % (E_me, names_ss_me))
        if i_me is None:
            raise RuntimeError('no combination has an entropy below +inf (k = {} exceeds '
                               'n_acc = {}, or the entropies are NaN)'.format(k, n_acc))

        # the parameters of the `closest' datasets, in accepted order
        thetas_closest = thetas[i_me, :n_closest]
        mrsses = dev.to_host(ops.mrsse(thetas, thetas_closest))
        MRSSE_min = np.inf
        names_ss_MRSSE = []
        set_ss_2stage = None
        for set_ss, names_ss, MRSSE_ss in zip(self.ss_candidates, names, mrsses):
            # If equal, dismiss the combination which contains uninformative summary statistics.
            if (MRSSE_ss == MRSSE_min and (len(names_ss_MRSSE) > len(names_ss))) \
                    or MRSSE_ss < MRSSE_min:
                MRSSE_min = MRSSE_ss
                names_ss_MRSSE = names_ss
                set_ss_2stage = set_ss
            logger.info('Combination %s shows the MRSSE of %f' % (names_ss, MRSSE_ss))
        logger.info('\nThe minimum MRSSE of %f was found in %s.' % (MRSSE_min, names_ss_MRSSE))
        self.scores = [dict(names=nm, entropy=float(e), mrsse=float(m))
                       for nm, e, m in zip(names, entropies, mrsses)]
        return set_ss_2stage

    # ---- the per-combination loop (any discrepancy) ----------------------------------------------
    def _obtain_accepted_thetas(self, set_ss, n_sim, n_acc, batch_size):
        """One rejection run with set_ss (diagnostics.py:172-212); the accepted parameters as a
        device (n_acc, q) array."""
        m = self.simulator.model.copy()
        list_ss = [em.Summary(ss, m[self.simulator.name], model=m) for ss in set_ss]
        if isinstance(self.fn_distance, str):
            d = em.Distance(self.fn_distance, *list_ss, model=m)
        else:
            d = em.Discrepancy(self.fn_distance, *list_ss, model=m)
        result = Rejection(d, batch_size=batch_size, seed=self.seed,
                           pool=self.pool).sample(n_acc, n_sim=n_sim)
        return _columns([result._dev[name] for name in result.parameter_names], n_acc)

    # ---- all combinations from one set of simulations ---------------------------------------------
    def _simulate(self, n_sim, batch_size):
        """The batches Rejection(..., batch_size, seed) runs for n_sim, each simulated once, with
        one Summary node per distinct candidate.  Returns the parameters (N, q) and summaries
        (N, W) on the device, the observed summaries (W,) and each candidate's column range."""
        m = self.simulator.model.copy()
        candidates = list(dict.fromkeys(ss for set_ss in self.ss_candidates for ss in set_ss))
        nodes = [em.Summary(ss, m[self.simulator.name], model=m).name for ss in candidates]
        params = m.parameter_names
        outputs = params + nodes + [em.observed_name(s) for s in nodes]
        plan = em.compile_plan(m, outputs)
        context = em.ComputationContext(batch_size=batch_size, seed=self.seed)
        n_batches = ceil(n_sim / batch_size)
        N = n_batches * batch_size
        P = S = obs = None
        ranges = {}
        for b in range(n_batches):
            batch = em.execute_batch(m, outputs, context, b, compiled=plan)
            context.num_submissions += 1
            theta = _columns([batch[p] for p in params], batch_size)
            sums = [_columns([batch[s]], batch_size) for s in nodes]
            if b == 0:
                obs_rows = [np.atleast_2d(dev.to_host(batch[em.observed_name(s)])) for s in nodes]
                col = 0
                for ss, o, x in zip(candidates, obs_rows, sums):
                    if o.shape != (1, x.shape[1]):
                        raise ValueError('the observed summary of {} has shape {}, its simulated '
                                         'rows {} columns'.format(ss.__name__, o.shape, x.shape[1]))
                    ranges[ss] = (col, int(x.shape[1]))
                    col += int(x.shape[1])
                obs = np.concatenate(obs_rows, axis=1).reshape(-1).astype(np.float64)
                P = dev.empty((N, int(theta.shape[1])))
                S = dev.empty((N, col))
            rows = slice(b * batch_size, (b + 1) * batch_size)
            P[rows] = theta
            for ss, x in zip(candidates, sums):
                c0, w = ranges[ss]
                S[rows, c0:c0 + w] = x
        return P, S, obs, ranges

    def _device_accepted_thetas(self, n_sim, n_acc, batch_size):
        """The accepted parameters (C, n_acc, q) of every combination from one simulation pass.

        Rejection's merge is a stable sort of [kept rows; batch rows] by distance (NaN last),
        batch after batch, so the rows it keeps are the first n_acc of one stable sort of all
        rows by distance in row order.  Here the same merge runs per combination over chunks of
        the resident rows, carrying the global row index, and the parameters are gathered once."""
        P, S, obs, ranges = self._simulate(n_sim, batch_size)
        N, q = int(P.shape[0]), int(P.shape[1])
        combs = [[ranges[ss] for ss in set_ss] for set_ss in self.ss_candidates]
        C = len(combs)
        # a block of (group combinations x chunk rows): whole columns while they fit, so that
        # each combination is merged once; rows are read once per group
        group = max(1, min(C, DISTANCE_BLOCK_BYTES // (8 * N)))
        chunk = max(1, min(N, DISTANCE_BLOCK_BYTES // (8 * group)))
        d = dev.empty((group, chunk))
        row_index = dev.to_device(np.arange(N, dtype=np.float64))
        rows = []
        for g0 in range(0, C, group):
            layout = ops.SubsetLayout(combs[g0:g0 + group], S.shape[1])
            ng = layout.n_combinations
            keys = [dev.empty((0,))] * ng
            kept = [dev.empty((0,))] * ng
            for r0 in range(0, N, chunk):
                nb = min(chunk, N - r0)
                ops.subset_distance(S[r0:r0 + nb], obs, layout, self.fn_distance,
                                    out=d[:ng, :nb])
                n_keep = min(n_acc, int(keys[0].shape[0]) + nb)
                for c in range(ng):
                    keys[c], kept[c] = ops.merge_topn([keys[c], kept[c]],
                                                      [d[c, :nb], row_index[r0:r0 + nb]],
                                                      keys[c], d[c, :nb], None, n_keep)
            rows += kept
        index = torch.stack(rows).reshape(-1).to(torch.int32)
        return ops.take_rows(P, index).reshape(C, n_acc, q)


def _columns(outputs, n):
    """np.column_stack of node outputs of n rows as a (n, width) float64 device matrix."""
    cols = []
    for x in outputs:
        t = x if dev.is_device_array(x) else dev.to_device(np.asarray(x, dtype=np.float64))
        if t.dtype != torch.float64:
            t = t.to(torch.float64)
        if t.dim() == 0 or t.dim() > 2 or t.shape[0] != n:
            raise ValueError('a summary or parameter output has shape {}; {} rows of at most '
                             'two axes were expected'.format(tuple(t.shape), n))
        cols.append(t if t.dim() == 2 else t[:, None])
    return torch.cat(cols, dim=1) if len(cols) > 1 else cols[0].contiguous()
