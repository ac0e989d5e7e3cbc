"""Array-level operators of the hot path: thin Python wrappers over the C ABI.

Each wrapper accepts CUDA tensors (or host arrays, which are uploaded) and returns CUDA
tensors.  Reference call sites are cited per function (paths relative to the reference repo).
"""
import ctypes

import numpy as np
import torch

from . import _lib
from . import device as dev

MAX_NESTED = _lib.CONSTANTS['MAX_NESTED']


def _matrix(S):
    if dev.is_device_array(S) and S.dtype == torch.float64 and S.dim() == 2 \
            and S.stride(1) == 1 and S.stride(0) >= S.shape[1]:
        return S  # row-strided views are consumed in place (leading dimension = stride(0))
    S = dev.to_device(S)
    if S.dim() == 1:
        S = S[:, None]
    if S.dim() != 2:
        raise ValueError('expected a 2-d (batch, dim) array, got shape {}'.format(tuple(S.shape)))
    if S.stride(1) != 1:
        S = S.contiguous()
    return S


def _ld(t):
    return t.stride(0) if t.shape[0] > 1 else t.shape[1]


def _out(out, shape, name):
    """A caller's ``out=`` for an entry point that writes rows of ``shape[1]`` adjacent doubles
    ``stride(0)`` apart (or, for a 1-d shape, one double per row): float64 device data of exactly
    ``shape`` whose rows do not overlap.  A transposed or column-strided view would be written in
    the wrong places, so it is refused."""
    if out is None:
        return dev.empty(shape)
    if not (dev.is_device_array(out) and out.dtype == torch.float64):
        raise ValueError('{}: out must be a float64 device tensor'.format(name))
    if tuple(out.shape) != tuple(shape):
        raise ValueError('{}: out must have shape {}, got {}'.format(name, tuple(shape),
                                                                     tuple(out.shape)))
    rows = shape[0]
    width = shape[1] if len(shape) > 1 else 1
    if (len(shape) > 1 and width > 1 and out.stride(1) != 1) or (rows > 1 and out.stride(0) < width):
        raise ValueError('{}: out must have unit column stride and non-overlapping rows, got '
                         'strides {}'.format(name, tuple(out.stride())))
    return out


def _params(params, model, names):
    """The (batch, p) parameter matrix of a model whose p parameters are ``names``."""
    P = _matrix(params)
    if P.shape[1] != len(names):
        raise ValueError('the {} model has {} parameters ({}), got a parameter width of {}'.format(
            model, len(names), ', '.join(names), P.shape[1]))
    return P


def _axes(x, name, layout):
    if x.dim() != len(layout) or any(isinstance(a, int) and a != n
                                     for a, n in zip(layout, x.shape)):
        raise ValueError('{} takes ({}) data, got shape {}'.format(
            name, ', '.join(str(a) for a in layout), tuple(x.shape)))
    return x


def _data(x, name, layout):
    """x as float64 device data with the axes ``layout`` (an int is a required size): device float64
    data is read in place, whatever its strides; anything else is uploaded."""
    if not (dev.is_device_array(x) and x.dtype == torch.float64):
        x = dev.to_device(x)
    return _axes(x, name, layout)


def _mask(x, name, layout):
    """x as bool or uint8 device data with the axes ``layout``, nonzero meaning set: such device
    data is read in place, whatever its strides; other device data is compared with 0, host data
    is uploaded first."""
    if not dev.is_device_array(x):
        x = dev.to_device(np.asarray(x, dtype=np.float64))
    if x.dtype not in (torch.bool, torch.uint8):
        x = x != 0
    return _axes(x, name, layout)


def _dist_obs(obs, D):
    """The observed row of a distance as a flat (D,) device vector."""
    obs_t = dev.to_device(obs).reshape(-1)
    if obs_t.numel() != D:
        raise ValueError('XA and XB must have the same number of columns '
                         '(i.e. feature dimension.)')
    return obs_t


def _dist_thresholds(thresholds, K, device_thresholds):
    """The K thresholds of a distance as a host float64 array (or None), or left as a contiguous
    float64 device tensor where the entry point reads them there (``device_thresholds``)."""
    thr = None
    if device_thresholds and dev.is_device_array(thresholds):
        thr = thresholds.reshape(-1)
        if thr.dtype != torch.float64 or not thr.is_contiguous():
            thr = thr.to(torch.float64).contiguous()
    elif thresholds is not None:
        thr = np.ascontiguousarray(np.atleast_1d(thresholds), dtype=np.float64)
    if thr is not None and thr.shape[0] != K:
        raise ValueError('need one threshold per distance column ({} != {})'.format(
            thr.shape[0], K))
    return thr


def _dist_prepare(S, obs, thresholds, K=1, want_indices=True, device_thresholds=False):
    """What the device distance wrappers share: the matrix, ``obs`` flattened and checked against
    its width, the K thresholds as a host float64 array (or None) -- or left as a device tensor
    where the entry point reads them there (``device_thresholds``) -- and the outputs d (B, K),
    acc_idx and n_acc (both None without thresholds)."""
    S = _matrix(S)
    B, D = S.shape
    obs_t = _dist_obs(obs, D)
    thr = _dist_thresholds(thresholds, K, device_thresholds)
    d = dev.empty((B, K))
    acc_idx = n_acc = None
    if thr is not None:
        n_acc = dev.zeros((1,), dtype=torch.int64)
        if want_indices:
            acc_idx = dev.empty((max(B, 1),), dtype=torch.int32)
    return S, obs_t, thr, d, acc_idx, n_acc


def _dist_accepted(acc_idx, n_acc, want_indices=True, sync=True):
    """What a distance wrapper returns next to d: None without thresholds, the pair
    (acc_idx, n_acc) left on the device when ``sync`` is False, else the accepted indices, or
    their number when the caller did not want indices."""
    if n_acc is None:
        return None
    if not sync:
        return acc_idx, n_acc
    n = int(n_acc.item())
    return acc_idx[:n] if want_indices else n


def dist_euclid(S, obs, w=None, thresholds=None, want_indices=True, sync=True, moments=False):
    """Euclidean / nested weighted distances of the rows of S to ``obs`` + acceptance.

    Replaces ``cdist(S, obs, 'euclidean'[, w=w])`` reached through
    elfi/model/utils.py:37-52 and elfi/model/elfi_model.py:1037, 1135-1151, and the mask of
    elfi/methods/inference/samplers.py:223-225.

    Parameters
    ----------
    S : (B, D) array
    obs : (D,) or (1, D) array
    w : None, (D,) or (K, D) -- cdist's ``w`` per nested column (a row of ones == unweighted)
    thresholds : None, float, (K,) host values, or a (K,) DEVICE array (no host round trip)
        -- accept rows with all_k(d[:, k] <= thresholds[k])
    sync : False leaves the accepted count on the device: acc_idx is then the pair
        (int32 buffer of B indices of which the first n_acc are valid, n_acc device int64[1])
    moments : True also returns the (2, D) device array [column means; column M2] of S, computed
        from the same read of S (AdaptiveDistance.add_data, elfi_model.py:1104-1125)

    Returns
    -------
    d : (B,) tensor if K == 1 and w was not 2-d, else (B, K)
    acc_idx : int32 tensor of accepted row indices, ascending (None without thresholds)
    """
    squeeze = True
    W = None
    K = 1
    if w is not None:
        W = dev.to_device(w)
        if W.dim() == 1:
            W = W[None, :]
        else:
            squeeze = False
        K = W.shape[0]
    S, obs_t, thr, d, acc_idx, n_acc = _dist_prepare(S, obs, thresholds, K, want_indices,
                                                     device_thresholds=True)
    B, D = S.shape
    if W is not None:
        if W.shape[1] != D:
            raise ValueError('weights must have {} columns'.format(D))
        if K > MAX_NESTED:
            raise ValueError('at most {} nested distances are supported'.format(MAX_NESTED))
    thr_on_device = dev.is_device_array(thr)
    mom = None
    if moments:
        mom = dev.empty((2, D))
        _lib.call('elfi_b200_dist_euclid_mom_f64', dev.context(), dev.ptr(S), _ld(S), B, D,
                  dev.ptr(obs_t), dev.ptr(W), K, None if thr_on_device else dev.ptr(thr),
                  dev.ptr(thr) if thr_on_device else None, dev.ptr(d), dev.ptr(acc_idx),
                  dev.ptr(n_acc), dev.ptr(mom), dev.stream_ptr())
    else:
        _lib.call('elfi_b200_dist_euclid_thr_dev_f64' if thr_on_device else
                  'elfi_b200_dist_euclid_thr_f64', dev.context(), dev.ptr(S), _ld(S), B, D,
                  dev.ptr(obs_t), dev.ptr(W), K, dev.ptr(thr), dev.ptr(d), dev.ptr(acc_idx),
                  dev.ptr(n_acc), dev.stream_ptr())
    acc_idx = _dist_accepted(acc_idx, n_acc, want_indices, sync)
    if squeeze:
        d = d.reshape(B)
    return (d, acc_idx, mom) if moments else (d, acc_idx)


# the header's ELFI_B200_METRIC_<NAME> codes by value: name -> code
_METRICS = {k[len('METRIC_'):].lower(): v for k, v in sorted(
    _lib.CONSTANTS.items(), key=lambda kv: kv[1]) if k.startswith('METRIC_')}
METRIC_CODES = {k: v for k, v in _METRICS.items() if k != 'euclidean'}


def dist_metric(S, obs, metric, p=2.0, threshold=None, want_indices=True):
    """cdist(S, obs, metric) for 'sqeuclidean', 'cityblock', 'chebyshev' and 'minkowski' (p)
    + acceptance, on the device (elfi/model/elfi_model.py:1016-1037 passes these metric strings to
    SciPy).  Minkowski with p = 1, 2, inf is routed to cityblock / euclidean / chebyshev as SciPy
    does.  Returns (d (B,), acc_idx or None)."""
    if metric == 'minkowski':
        if p == 1:
            metric = 'cityblock'
        elif p == 2:
            return dist_euclid(S, obs, thresholds=threshold, want_indices=want_indices)
        elif np.isinf(p):
            metric = 'chebyshev'
        elif not p > 0:
            raise ValueError('p must be greater than 0')
    if metric not in METRIC_CODES:
        raise ValueError('Unknown Distance Metric: {}'.format(metric))
    S, obs_t, thr, d, acc_idx, n_acc = _dist_prepare(S, obs, threshold, 1, want_indices)
    B, D = S.shape
    _lib.call('elfi_b200_dist_metric_thr_f64', dev.context(), METRIC_CODES[metric], float(p),
              dev.ptr(S), _ld(S), B, D, dev.ptr(obs_t), dev.ptr(thr), dev.ptr(d), dev.ptr(acc_idx),
              dev.ptr(n_acc), dev.stream_ptr())
    return d.reshape(B), _dist_accepted(acc_idx, n_acc, want_indices)


def dist_seuclidean(S, obs, V, threshold=None, want_indices=True):
    """cdist(S, obs, 'seuclidean', V=V) + acceptance on the device, bit-identical to SciPy (two
    running sums and an IEEE division per term; elfi/model/elfi_model.py:1016-1037 forwards the
    metric string and V to cdist).  Returns (d (B,), acc_idx or None)."""
    S, obs_t, thr, d, acc_idx, n_acc = _dist_prepare(S, obs, threshold, 1, want_indices)
    B, D = S.shape
    V_t = dev.to_device(V)
    if V_t.dim() != 1 or V_t.shape[0] != D:
        raise ValueError('Variance vector V must be of the same dimension as the vectors on '
                         'which the distances are computed.')
    _lib.call('elfi_b200_dist_seuclidean_thr_f64', dev.context(), dev.ptr(S), _ld(S), B, D,
              dev.ptr(obs_t), dev.ptr(V_t), dev.ptr(thr), dev.ptr(d), dev.ptr(acc_idx),
              dev.ptr(n_acc), dev.stream_ptr())
    return d.reshape(B), _dist_accepted(acc_idx, n_acc, want_indices)


MAHALANOBIS_D_MAX = _lib.CONSTANTS['MAHALANOBIS_D_MAX']


def dist_mahalanobis(S, obs, VI, threshold=None, want_indices=True):
    """cdist(S, obs, 'mahalanobis', VI=VI) + acceptance on the device, bit-identical to SciPy for
    any (D, D) VI (t = VI u by rows of VI, then u . t, both in SciPy's two-sum order;
    elfi/model/elfi_model.py:1016-1037 forwards the metric string and VI to cdist).  D is at most
    MAHALANOBIS_D_MAX.  Returns (d (B,), acc_idx or None)."""
    S, obs_t, thr, d, acc_idx, n_acc = _dist_prepare(S, obs, threshold, 1, want_indices)
    B, D = S.shape
    if D > MAHALANOBIS_D_MAX:
        raise ValueError('dist_mahalanobis: D={} is above MAHALANOBIS_D_MAX = {}'.format(
            D, MAHALANOBIS_D_MAX))
    VI_t = dev.to_device(VI)
    if tuple(VI_t.shape) != (D, D):
        raise ValueError('VI must be a ({0}, {0}) matrix for summaries of dimension {0}, got shape '
                         '{1}'.format(D, tuple(VI_t.shape)))
    _lib.call('elfi_b200_dist_mahalanobis_thr_f64', dev.context(), dev.ptr(S), _ld(S), B, D,
              dev.ptr(obs_t), dev.ptr(VI_t), dev.ptr(thr), dev.ptr(d), dev.ptr(acc_idx),
              dev.ptr(n_acc), dev.stream_ptr())
    return d.reshape(B), _dist_accepted(acc_idx, n_acc, want_indices)


def autocov(x, lags=(1,), out=None):
    """MA2 autocovariance summaries (elfi/examples/ma2.py:40-59) for one or more lags.

    Returns a (B, len(lags)) tensor: column l is ``np.mean(x[:, lag:] * x[:, :-lag], axis=1)``
    bit for bit.  This is already the column-stacked summary matrix of
    elfi/model/utils.py:39, so it can be handed to :func:`dist_euclid` directly."""
    x = _matrix(x)
    B, n = x.shape
    lags_arr = np.ascontiguousarray(np.atleast_1d(lags), dtype=np.int32)
    for lag in lags_arr:
        if not 1 <= lag < n:
            raise ValueError('lag {} outside [1, {})'.format(lag, n))
    out = _out(out, (B, len(lags_arr)), 'autocov')
    _lib.call('elfi_b200_summary_autocov_f64', dev.context(), dev.ptr(x), _ld(x), B, n,
              dev.ptr(lags_arr), len(lags_arr), dev.ptr(out), out.stride(0) if B > 1 else
              out.shape[1], dev.stream_ptr())
    return out


def meanvar(y, out=None):
    """Gaussian-model summaries ss_mean / ss_var (elfi/examples/gauss.py:142-173).

    Returns a (B, 2) tensor [np.mean(y, axis=1), np.var(y, axis=1)], bit for bit."""
    y = _matrix(y)
    B, n = y.shape
    out = _out(out, (B, 2), 'meanvar')
    _lib.call('elfi_b200_summary_meanvar_f64', dev.context(), dev.ptr(y), _ld(y), B, n,
              dev.ptr(out), out.stride(0) if B > 1 else out.shape[1], 0, 1, dev.stream_ptr())
    return out


def argsort(keys, return_keys=False):
    """Stable ascending argsort of a 1-d fp64 array (NaN last) -> int32 permutation.

    np.argsort of elfi/methods/inference/samplers.py:235 and elfi/methods/utils.py:397."""
    keys = dev.to_device(keys).reshape(-1)
    n = keys.numel()
    perm = dev.empty((n,), dtype=torch.int32)
    ks = dev.empty((n,)) if return_keys else None
    _lib.call('elfi_b200_sort_pairs_f64', dev.context(), dev.ptr(keys), n, dev.ptr(ks),
              dev.ptr(perm), dev.stream_ptr())
    return (perm, ks) if return_keys else perm


def _as_2d(t):
    if t.dim() == 2:
        return t
    width = 1
    for extent in t.shape[1:]:
        width *= int(extent)
    return t.reshape(t.shape[0], width)


def take_rows(src, idx):
    """src[idx] for an fp64 array with the batch on axis 0 (samplers.py:230, 237)."""
    src = dev.to_device(src)
    shape = src.shape
    s2 = _as_2d(src)
    if s2.stride(-1) != 1 and s2.shape[1] > 0:
        s2 = s2.contiguous()
    idx = dev.to_device(idx, dtype=torch.int32)
    n = idx.numel()
    width = s2.shape[1]
    dst = dev.empty((n, width))
    if n and width:
        _lib.call('elfi_b200_gather_rows_f64', dev.context(), dev.ptr(s2), _ld(s2), dev.ptr(idx),
                  n, width, dev.ptr(dst), width, dev.stream_ptr())
    return dst.reshape((n,) + tuple(shape[1:]))


def merge_topn(state, batch, key_state, key_batch, map_b, n_keep):
    """Rejection._merge_batch (samplers.py:226-237) as one library call: the virtual concatenation
    [state[k]; batch[k][map_b]] is ranked by [key_state; key_batch[map_b]] (1-d views, possibly a
    strided column of a (rows, K) distance matrix) and the n_keep smallest rows of every output k
    come back as new device arrays.  map_b None: every batch row is a candidate."""
    if map_b is not None and map_b.dtype != torch.int32:
        raise TypeError('map_b must be an int32 device array of batch row indices')
    n_a = int(key_state.shape[0])
    n_b = int(map_b.numel()) if map_b is not None else int(key_batch.shape[0])
    a2 = [_as_2d(t) for t in state]
    b2 = [_as_2d(dev.to_device(t)) for t in batch]
    widths = [t.shape[1] for t in b2]
    outs = [dev.empty((n_keep, w)) for w in widths]
    n = len(outs)
    if n_keep and n:
        arr_p, arr_i = ctypes.c_void_p * n, ctypes.c_int64 * n
        pa = arr_p(*[t.data_ptr() if n_a else 0 for t in a2])
        la = arr_i(*[_ld(t) if n_a else w for t, w in zip(a2, widths)])
        pb = arr_p(*[t.data_ptr() for t in b2])
        lb = arr_i(*[_ld(t) for t in b2])
        wd = arr_i(*widths)
        pd = arr_p(*[t.data_ptr() for t in outs])
        ld = arr_i(*widths)
        cast = lambda a: ctypes.cast(a, ctypes.c_void_p)   # noqa: E731
        _lib.call('elfi_b200_topn_merge_f64', dev.context(), dev.ptr(key_state) if n_a else None,
                  key_state.stride(0) if n_a > 1 else 1, n_a, dev.ptr(key_batch),
                  key_batch.stride(0) if key_batch.shape[0] > 1 else 1, dev.ptr(map_b), n_b,
                  n_keep, n, cast(pa), cast(la), cast(pb), cast(lb), cast(wd), cast(pd), cast(ld),
                  dev.stream_ptr())
    return [o.reshape((n_keep,) + tuple(t.shape[1:])) for o, t in zip(outs, batch)]


def _seg_rows(t, R):
    """(R, rows, width) view of a segmented device array (R, rows, *shape), in place when its
    trailing dimensions are contiguous: (pointer, leading dimension, segment stride, width)."""
    if t.dim() < 2 or t.shape[0] != R:
        raise ValueError('expected an (R={}, rows, ...) array, got shape {}'.format(
            R, tuple(t.shape)))
    rows = int(t.shape[1])
    width = 1
    for extent in t.shape[2:]:
        width *= int(extent)
    v = t.reshape(R, rows, width)
    if v.stride(2) != 1 and width > 1:
        v = v.contiguous()
    ld = v.stride(1) if rows > 1 else width
    return v, ld, v.stride(0), width


def merge_topn_seg(state, batch, key_state, key_batch, n_keep):
    """R independent :func:`merge_topn` calls (map_b None) in one library call: segment r ranks
    [state[k][r]; batch[k][r]] by [key_state[r]; key_batch[r]] and keeps its n_keep smallest rows.
    state[k] is (R, nA, ...), batch[k] (R, nB, ...), key_state (R, nA) and key_batch (R, nB) (views
    such as a column of a distance matrix are read in place).  Returns new (R, n_keep, ...) device
    arrays, each segment bit-identical to merge_topn on that segment."""
    R = int(key_batch.shape[0])
    n_a, n_b = int(key_state.shape[1]), int(key_batch.shape[1])
    a3 = [_seg_rows(t, R) for t in state]
    b3 = [_seg_rows(dev.to_device(t), R) for t in batch]
    widths = [w for _, _, _, w in b3]
    outs = [dev.empty((R, n_keep, w)) for w in widths]
    n = len(outs)
    if n_keep and n:
        arr_p, arr_i = ctypes.c_void_p * n, ctypes.c_int64 * n
        pa = arr_p(*[v.data_ptr() if n_a else 0 for v, _, _, _ in a3])
        la = arr_i(*[ld if n_a else w for (_, ld, _, _), w in zip(a3, widths)])
        sa = arr_i(*[s for _, _, s, _ in a3])
        pb = arr_p(*[v.data_ptr() for v, _, _, _ in b3])
        lb = arr_i(*[ld for _, ld, _, _ in b3])
        sb = arr_i(*[s for _, _, s, _ in b3])
        wd = arr_i(*widths)
        pd = arr_p(*[t.data_ptr() for t in outs])
        ld = arr_i(*widths)
        sd = arr_i(*[n_keep * w for w in widths])
        cast = lambda a: ctypes.cast(a, ctypes.c_void_p)   # noqa: E731
        _lib.call('elfi_b200_topn_merge_seg_f64', dev.context(), R,
                  dev.ptr(key_state) if n_a else None, key_state.stride(1) if n_a > 1 else 1,
                  key_state.stride(0) if n_a else 0, n_a, dev.ptr(key_batch),
                  key_batch.stride(1) if n_b > 1 else 1, key_batch.stride(0), n_b, n_keep, n,
                  cast(pa), cast(la), cast(sa), cast(pb), cast(lb), cast(sb), cast(wd), cast(pd),
                  cast(ld), cast(sd), dev.stream_ptr())
    return [o.reshape((R, n_keep) + tuple(t.shape[2:])) for o, t in zip(outs, batch)]


SEG_METRICS = ('euclidean', 'sqeuclidean', 'cityblock', 'chebyshev', 'minkowski')


def dist_seg(S, obs, metric='euclidean', p=2.0):
    """Segmented distances: S (R B, D) in R segments of B rows, segment r against observed row r
    of obs (R, D); returns d (R B,).  Each segment is bit-identical to dist_euclid (unweighted) or
    dist_metric on that segment; Minkowski with p = 1, 2, inf is routed as dist_metric does."""
    if metric == 'minkowski':
        if p == 1:
            metric = 'cityblock'
        elif p == 2:
            metric = 'euclidean'
        elif np.isinf(p):
            metric = 'chebyshev'
        elif not p > 0:
            raise ValueError('p must be greater than 0')
    if metric not in SEG_METRICS:
        raise ValueError('dist_seg supports {}, not {!r}'.format(', '.join(SEG_METRICS), metric))
    code = 0 if metric == 'euclidean' else METRIC_CODES[metric]
    S = _matrix(S)
    O = _matrix(obs)
    R, D = O.shape
    n = S.shape[0]
    if S.shape[1] != D:
        raise ValueError('XA and XB must have the same number of columns '
                         '(i.e. feature dimension.)')
    if n % R:
        raise ValueError('{} rows do not form {} equal segments'.format(n, R))
    d = dev.empty((n,))
    _lib.call('elfi_b200_dist_seg_f64', dev.context(), code, float(p), dev.ptr(S), _ld(S), R,
              n // R, D, dev.ptr(O), _ld(O), dev.ptr(d), dev.stream_ptr())
    return d


class CandidateBuffer:
    """Packed (capacity, width) device buffer of accepted rows + device-side row count: the tail
    of the reference's sample buffers (samplers.py:196-230) filled without host round trips."""

    def __init__(self, capacity, widths):
        self.widths = [int(w) for w in widths]
        self.width = sum(self.widths)
        self.capacity = int(capacity)
        self.rows = dev.empty((self.capacity, self.width))
        self._counters = dev.zeros((2,), dtype=torch.int64)      # [count, dropped]: one D2H reads both
        self.count = self._counters[0:1]
        self.dropped = self._counters[1:2]

    def reset(self):
        self._counters.zero_()

    @staticmethod
    def _rows(sources):
        """The sources as (B, width) views; the append reads width adjacent doubles per row, so a
        view whose columns are not adjacent would be read in the wrong places and is refused."""
        srcs = [_as_2d(t) for t in sources]
        for t in srcs:
            if t.shape[1] > 1 and t.stride(1) != 1:
                raise ValueError('sources must have unit column stride, got strides {}'.format(
                    tuple(t.stride())))
        return srcs

    def _descriptors(self, sources):
        """ctypes descriptor arrays of a source list, cached while the same buffers come back
        (a sampler appends from the same output tensors batch after batch)."""
        key = tuple((t.data_ptr(), tuple(t.shape), tuple(t.stride())) for t in sources)
        cached = getattr(self, '_desc', None)
        if cached is not None and cached[0] == key:
            return cached[1]
        srcs = self._rows(sources)
        if [t.shape[1] for t in srcs] != self.widths:
            raise ValueError('source widths do not match the buffer layout')
        n = len(srcs)
        ptrs = (ctypes.c_void_p * n)(*[t.data_ptr() for t in srcs])
        lds = (ctypes.c_int64 * n)(*[_ld(t) for t in srcs])
        wid = (ctypes.c_int64 * n)(*self.widths)
        desc = (n, ptrs, lds, wid, ctypes.cast(ptrs, ctypes.c_void_p),
                ctypes.cast(lds, ctypes.c_void_p), ctypes.cast(wid, ctypes.c_void_p),
                dev.ptr(self.rows), dev.ptr(self.count), dev.ptr(self.dropped))
        self._desc = (key, desc)
        return desc

    def append(self, sources, acc_idx, n_acc, max_rows):
        """Append rows acc_idx[:n_acc] (device int32 / device int64 count) of `sources`."""
        n, _, _, _, pp, pl, pw, prow, pcount, pdrop = self._descriptors(sources)
        _lib.call('elfi_b200_accept_append_f64', dev.context(), dev.ptr(acc_idx), dev.ptr(n_acc),
                  int(max_rows), n, pp, pl, pw, prow, self.width, self.capacity, pcount, pdrop,
                  dev.stream_ptr())

    def bind_batch(self, S, obs, thresholds, d_out, acc_idx, n_acc, extras, w=None):
        """A zero-argument callable running ONE threshold-mode batch -- distances of S + acceptance
        + append of the accepted rows [d | extras] to this buffer -- as a single library call
        (elfi_b200_rejection_batch_f64) with every argument marshalled once: microseconds of host
        time per batch, so that a busy host cannot starve a sub-millisecond kernel.  All tensors are device
        tensors the caller keeps alive; `thresholds` is a host sequence or a device tensor of K
        float64 values (read at every call, so it may be updated in place between calls)."""
        S = _matrix(S)
        B, D = S.shape
        W = None if w is None else dev.to_device(w).reshape(-1, D)
        K = 1 if W is None else W.shape[0]
        extras = self._rows(extras)
        if [K] + [t.shape[1] for t in extras] != self.widths:
            raise ValueError('d / extra widths do not match the buffer layout')
        if thresholds is None:
            raise ValueError('bind_batch needs thresholds (a host sequence or a device tensor)')
        thr_dev = thresholds if dev.is_device_array(thresholds) else None
        if thr_dev is not None and not (thr_dev.dtype == torch.float64 and thr_dev.is_contiguous()):
            raise ValueError('device thresholds must be a contiguous float64 tensor (a converted '
                             'copy would not see updates made in place)')
        thr_host = None if thr_dev is not None else np.ascontiguousarray(
            np.atleast_1d(thresholds), dtype=np.float64)
        n_thr = thr_dev.numel() if thr_dev is not None else thr_host.size
        if n_thr != K:
            raise ValueError('need one threshold per distance column ({} != {})'.format(n_thr, K))
        n = len(extras)
        ptrs = (ctypes.c_void_p * max(n, 1))(*[t.data_ptr() for t in extras])
        lds = (ctypes.c_int64 * max(n, 1))(*[_ld(t) for t in extras])
        wid = (ctypes.c_int64 * max(n, 1))(*[t.shape[1] for t in extras])
        keep = (S, obs, W, thr_dev, thr_host, d_out, acc_idx, n_acc, extras, ptrs, lds, wid)
        args = (dev.context(), dev.ptr(S), S.stride(0) if B > 1 else D, B, D, dev.ptr(obs),
                dev.ptr(W), K, dev.ptr(thr_host), dev.ptr(thr_dev), dev.ptr(d_out),
                dev.ptr(acc_idx), dev.ptr(n_acc), n, ctypes.cast(ptrs, ctypes.c_void_p),
                ctypes.cast(lds, ctypes.c_void_p), ctypes.cast(wid, ctypes.c_void_p),
                dev.ptr(self.rows), self.width, self.capacity, dev.ptr(self.count),
                dev.ptr(self.dropped))

        def run(_keep=keep):
            _lib.call('elfi_b200_rejection_batch_f64', *args, dev.stream_ptr())
        return run

    def best(self, n, key_col=None):
        """(rows sorted by column key_col, first n; count, dropped) -- one D2H of the counters.

        The default key is the last column of the first source, the distance block: the
        reference ranks nested distances by their last column (samplers.py:231-233).  Ties keep
        the order in which the rows were appended."""
        if key_col is None:
            key_col = self.widths[0] - 1
        count, dropped = (int(v) for v in self._counters.cpu().tolist())
        keys = self.rows[:count, key_col].contiguous()
        perm = argsort(keys)
        return take_rows(self.rows, perm[:min(n, count)]), count, dropped


def weighted_sample_quantile(x, alpha, weights=None):
    """elfi/methods/utils.py:379-411 on the device; returns a Python float."""
    x = dev.to_device(x).reshape(-1)
    w = None if weights is None else dev.to_device(weights).reshape(-1)
    if w is not None and w.numel() != x.numel():
        raise ValueError('x and weights must have the same length')
    out = dev.empty((2,))
    _lib.call('elfi_b200_wquantile_f64', dev.context(), dev.ptr(x), dev.ptr(w), x.numel(),
              float(alpha), dev.ptr(out), dev.stream_ptr())
    return float(out[0].item())


def colmoments(S):
    """(mean, M2) per column of one batch (AdaptiveDistance.add_data's per-batch ingredients,
    elfi/model/elfi_model.py:1104-1125).  Returns two host arrays of length D."""
    S = _matrix(S)
    B, D = S.shape
    out = dev.empty((2, D))
    _lib.call('elfi_b200_colmoments_f64', dev.context(), dev.ptr(S), _ld(S), B, D, dev.ptr(out),
              dev.stream_ptr())
    out = out.cpu().numpy()
    return out[0], out[1]


def weighted_stats(x, weights=None):
    """V1, V2, weighted mean and unbiased weighted variance (elfi/methods/utils.py:108-139).

    Returns (V1, V2, xbar (p,), s2 (p,)) as host values."""
    x = _matrix(x)
    N, p = x.shape
    w = None if weights is None else dev.to_device(weights).reshape(-1)
    stats = dev.empty((2 + 2 * p,))
    _lib.call('elfi_b200_weighted_stats_f64', dev.context(), dev.ptr(x), _ld(x), dev.ptr(w), N, p,
              dev.ptr(stats), dev.stream_ptr())
    s = stats.cpu().numpy()
    return s[0], s[1], s[2:2 + p].copy(), s[2 + p:2 + 2 * p].copy()


def weighted_var(x, weights=None):
    """elfi/methods/utils.py:108-139."""
    return weighted_stats(x, weights)[3]


def gm_logpdf(x, means, cov=1, weights=None, validate=True, mixed=False):
    """GMDistribution.logpdf (elfi/methods/utils.py:174-197) on the device.

    x (N, p) and means (M, p) may be host or device arrays; returns a device tensor (N,).
    ``validate=False`` skips the two synchronising weight checks of normalize_weights
    (utils.py:80-88) for weights the caller produced itself.  ``mixed=True`` takes 2^f from the
    fp32 special-function unit (term error <= 2.5e-7 instead of 1.9e-9, fewer fp64 instructions
    per term): the throughput
    mode's choice, where parity with the reference is statistical."""
    means = _matrix(means)
    M, p = means.shape
    x = dev.to_device(x)
    x = x.reshape(-1, p) if x.dim() != 2 else x
    x = _matrix(x)
    N = x.shape[0]
    cov = np.atleast_2d(np.asarray(cov, dtype=np.float64))
    if cov.shape == (1, 1) and p > 1:
        cov = np.eye(p) * cov[0, 0]
    L = np.linalg.cholesky(cov)
    Linv = np.ascontiguousarray(np.linalg.inv(L))
    logdet = 2.0 * float(np.sum(np.log(np.diag(L))))
    w = None if weights is None else dev.to_device(weights).reshape(-1)
    if w is not None and validate:
        if bool((w < 0).any()):
            raise ValueError("Weights must be positive")
        if float(w.sum()) == 0:
            raise ValueError("All weights are zero")
    logq = dev.empty((N,))
    _lib.call('elfi_b200_gm_logpdf_mixed_f64' if mixed else 'elfi_b200_gm_logpdf_f64',
              dev.context(), dev.ptr(x), _ld(x), N, dev.ptr(means),
              _ld(means), dev.ptr(w), M, p, dev.ptr(Linv), logdet, dev.ptr(logq), dev.stream_ptr())
    return logq


def smc_weights(logprior, logq):
    """w = exp(logprior - logq) (elfi/methods/inference/samplers.py:514)."""
    lp = dev.to_device(logprior).reshape(-1)
    lq = dev.to_device(logq).reshape(-1)
    w = dev.empty((lp.numel(),))
    _lib.call('elfi_b200_smc_weights_f64', dev.context(), dev.ptr(lp), dev.ptr(lq), lp.numel(),
              dev.ptr(w), dev.stream_ptr())
    return w


# ------------------------------------------------------------------ throughput mode (device RNG)
def prior_ma2(batch_size, seed, offset=0, t1=None, which='both'):
    """MA2 prior draws on the device (elfi/examples/ma2.py:96-186).

    which='both' -> (t1, t2); 't1' -> t1; 't2' -> t2 conditional on the given t1."""
    mode = {'both': 0, 't1': 1, 't2': 2}[which]
    if mode == 2:
        t1 = dev.to_device(t1).reshape(-1).contiguous()
        batch_size = t1.numel()
    else:
        t1 = dev.empty((batch_size,))
    t2 = dev.empty((batch_size,)) if mode != 1 else None
    _lib.call('elfi_b200_prior_ma2_f64', dev.context(), batch_size, int(seed), int(offset), mode,
              dev.ptr(t1), dev.ptr(t2), dev.stream_ptr())
    return (t1, t2) if mode == 0 else (t1 if mode == 1 else t2)


def logprior_ma2(params):
    """Joint log prior density of MA2's (t1, t2); -inf outside the support."""
    x = _matrix(params)
    out = dev.empty((x.shape[0],))
    _lib.call('elfi_b200_logprior_ma2_f64', dev.context(), dev.ptr(x), _ld(x), x.shape[0],
              dev.ptr(out), dev.stream_ptr())
    return out


def sim_ma2(t1, t2, n_obs=100, seed=0, offset=0, want_data=False, want_summaries=True):
    """MA2 simulator on the device; returns (X or None, S or None) with S = autocov lags (1, 2)
    computed in the same kernel (X never touches HBM unless asked for)."""
    t1 = dev.to_device(t1).reshape(-1)
    t2 = dev.to_device(t2).reshape(-1)
    B = t1.numel()
    X = dev.empty((B, n_obs)) if want_data else None
    S = dev.empty((B, 2)) if want_summaries else None
    _lib.call('elfi_b200_sim_ma2_f64', dev.context(), dev.ptr(t1), dev.ptr(t2), B, n_obs,
              int(seed), int(offset), dev.ptr(X), n_obs, dev.ptr(S), 2, dev.stream_ptr())
    return X, S


def gm_cdf(weights, n=None):
    """Inclusive running sum of the mixture weights (None -> n equal weights): the lookup table of
    the component draw in GMDistribution.rvs (elfi/methods/utils.py:239), built once per population
    and handed to every :func:`gm_rvs` call of that population."""
    w = None if weights is None else dev.to_device(weights).reshape(-1)
    n = int(w.numel()) if w is not None else int(n)
    cumw = dev.empty((n,))
    _lib.call('elfi_b200_gm_cdf_f64', dev.context(), dev.ptr(w), n, dev.ptr(cumw), dev.stream_ptr())
    return cumw


def gm_rvs(means, cov, weights, size, seed, offset=0, support=0, box=None, cdf=None, prior=None,
           sources=None):
    """GMDistribution.rvs on the device (elfi/methods/utils.py:200-261) for p <= 16; support=1
    keeps only draws inside the MA2 prior support, support=2 inside ``box`` = (lo (p,), hi (p,)),
    support=3 where the joint log density of ``prior`` (a (p, 5) table of :func:`prior_logpdf`) is
    finite (redrawn per particle), support=4 the same with conditional priors (``sources`` (p, 2)
    as in :func:`prior_logpdf`; the draws of support 3 when every source is -1).  ``cdf`` =
    :func:`gm_cdf` of the weights (then ``weights`` is not read)."""
    means = _matrix(means)
    N, p = means.shape
    cov = np.atleast_2d(np.asarray(cov, dtype=np.float64))
    if cov.shape == (1, 1) and p > 1:
        cov = np.eye(p) * cov[0, 0]
    L = np.ascontiguousarray(np.linalg.cholesky(cov))
    boxarr = None
    if support == 2:
        boxarr = np.ascontiguousarray(np.concatenate([np.asarray(box[0], dtype=np.float64),
                                                      np.asarray(box[1], dtype=np.float64)]))
    elif support in (3, 4):
        boxarr = _prior_table(prior, sources if support == 4 else None)
        if support == 4 and sources is None:
            raise ValueError('support 4 takes the sources of the conditional priors')
        if boxarr.shape[0] != p:
            raise ValueError('the prior table has {} parameters, the mixture {}'.format(
                boxarr.shape[0], p))
    out = dev.empty((size, p))
    if cdf is None:
        cdf = gm_cdf(weights, N)
    elif cdf.numel() != N:
        raise ValueError('cdf must have one entry per mixture component')
    _lib.call('elfi_b200_gm_rvs_cdf_f64', dev.context(), dev.ptr(means), _ld(means), dev.ptr(cdf), N,
              p, dev.ptr(L), size, int(seed), int(offset), int(support), dev.ptr(boxarr),
              dev.ptr(out), p, dev.stream_ptr())
    return out


# stock scipy.stats priors: a parameter is [kind, p0, p1, p2, p3], scipy's positional parameters
# with loc and scale filled in (include/elfi_b200.h; elfi_b200.priors builds them from a model)
PRIOR_KINDS = ('uniform', 'norm', 'truncnorm', 'expon', 'gamma', 'beta')
PRIOR_SHAPES = {'uniform': (), 'norm': (), 'truncnorm': ('a', 'b'), 'expon': (), 'gamma': ('a',),
                'beta': ('a', 'b')}
MAX_PRIOR_PARAMS = _lib.CONSTANTS['MAX_PRIOR_PARAMS']
PRIOR_SPEC_WORDS = _lib.CONSTANTS['PRIOR_SPEC_WORDS']
PRIOR_COND_SPEC_WORDS = _lib.CONSTANTS['PRIOR_COND_SPEC_WORDS']


def _prior_spec_error(spec, loc_src=-1, scale_src=-1):
    """Why a [kind, p0, p1, p2, p3] row is invalid (the library's checks), or None.  A loc or
    scale with a source (>= 0) is a placeholder and is not checked."""
    k = spec[0]
    if k not in range(len(PRIOR_KINDS)):
        return 'unknown kind {!r} (supported: {})'.format(k, ', '.join(PRIOR_KINDS))
    name = PRIOR_KINDS[int(k)]
    ns = len(PRIOR_SHAPES[name])
    shapes = spec[1:1 + ns]
    loc = spec[1 + ns] if loc_src < 0 else 0.0
    scale = spec[2 + ns] if scale_src < 0 else 1.0
    if not (np.isfinite(loc) and np.isfinite(scale) and scale > 0):
        return 'loc must be finite and scale finite and > 0 (loc {}, scale {})'.format(loc, scale)
    if name == 'truncnorm' and not shapes[0] < shapes[1]:
        return 'truncnorm needs a < b (a {}, b {})'.format(*shapes)
    if name in ('gamma', 'beta') and not all(np.isfinite(s) and s > 0 for s in shapes):
        return '{} needs finite shape parameters > 0 ({})'.format(name, ', '.join(
            '{} {}'.format(n, s) for n, s in zip(PRIOR_SHAPES[name], shapes)))
    return None


def _prior_sources(sources, p):
    """(p, 2) float64 [loc_src, scale_src] per parameter: -1 or another column 0 <= j < p."""
    s = np.asarray(sources, dtype=np.float64)
    if s.shape != (p, 2):
        raise ValueError('sources are (p, 2) = ({}, 2) [loc_src, scale_src], got shape {}'.format(
            p, s.shape))
    for a in range(p):
        for w, what in enumerate(('loc', 'scale')):
            v = s[a, w]
            if not (v == -1 or (0 <= v < p and v == int(v) and v != a)):
                raise ValueError('prior parameter {}: the {} source must be -1 or a column '
                                 '0 <= j < {} other than {}, got {}'.format(a, what, p, a, v))
    return s


def _prior_table(specs, sources=None):
    """The (p, 5) table, or with sources the (p, 7) table of conditional priors."""
    t = np.ascontiguousarray(np.atleast_2d(np.asarray(specs, dtype=np.float64)))
    if t.ndim != 2 or t.shape[1] != 5 or not 1 <= t.shape[0] <= MAX_PRIOR_PARAMS:
        raise ValueError('a prior table is (p, 5) with 1 <= p <= {}, got shape {}'.format(
            MAX_PRIOR_PARAMS, np.shape(specs)))
    src = None if sources is None else _prior_sources(sources, t.shape[0])
    for i, row in enumerate(t):
        why = _prior_spec_error(row, *(() if src is None else src[i]))
        if why:
            raise ValueError('prior parameter {}: {}'.format(i, why))
    return t if src is None else np.ascontiguousarray(np.concatenate([t, src], axis=1))


def _row_vector(v, size, what):
    if v is None:
        return None
    v = dev.to_device(v).reshape(-1)
    if v.numel() == 1 and size != 1:
        v = v.expand(size)
    if v.numel() != size:
        raise ValueError('{} has {} values for {} draws'.format(what, v.numel(), size))
    return v.contiguous()


def prior_rvs(spec, size, seed, offset=0, loc=None, scale=None):
    """``size`` draws of one stock prior on the device: spec = [kind, p0, p1, p2, p3]
    (PRIOR_KINDS, scipy's positional parameters).  Row i is a pure function of (seed, offset + i).
    ``loc`` / ``scale``: per-row values (size,) that replace spec's (then its word is a
    placeholder), for a prior whose loc or scale is another parameter; draw i is then loc_i +
    scale_i y_i with y_i the standard draw of the same stream, NaN where scale_i < 0 or NaN.
    Returns a device tensor (size,)."""
    size = int(size)
    t = np.ascontiguousarray(np.atleast_2d(np.asarray(spec, dtype=np.float64)))
    if t.shape[0] != 1:
        raise ValueError('prior_rvs draws one parameter; got {} specs'.format(t.shape[0]))
    lv, sv = _row_vector(loc, size, 'loc'), _row_vector(scale, size, 'scale')
    if t.shape[1] == 5:
        why = _prior_spec_error(t[0], -1 if lv is None else 0, -1 if sv is None else 0)
        if why:
            raise ValueError('prior parameter 0: ' + why)
    else:
        _prior_table(t)                     # the shape error
    out = dev.empty((size,))
    if lv is None and sv is None:
        _lib.call('elfi_b200_prior_rvs_f64', dev.context(), dev.ptr(t), size, int(seed),
                  int(offset), dev.ptr(out), dev.stream_ptr())
    else:
        _lib.call('elfi_b200_prior_rvs_cond_f64', dev.context(), dev.ptr(t), size, int(seed),
                  int(offset), dev.ptr(lv), dev.ptr(sv), dev.ptr(out), dev.stream_ptr())
    return out


def prior_logpdf(params, specs, sources=None):
    """Joint log density of independent stock priors at the rows of params (B, p): the sum, left
    to right, of scipy.stats.<kind>.logpdf per column; -inf outside the support.  specs (p, 5).
    ``sources`` (p, 2) [loc_src, scale_src]: -1 for the table's constant, j for column j of the
    same row (a conditional prior; include/elfi_b200.h has the per-row rule).  Returns a device
    tensor (B,)."""
    t = _prior_table(specs, sources)
    x = _matrix(params)
    if x.shape[1] != t.shape[0]:
        raise ValueError('params have {} columns, the prior table {} rows'.format(x.shape[1],
                                                                                 t.shape[0]))
    out = dev.empty((x.shape[0],))
    name = 'elfi_b200_prior_logpdf_f64' if sources is None else 'elfi_b200_prior_logpdf_cond_f64'
    _lib.call(name, dev.context(), dev.ptr(x), _ld(x), x.shape[0], t.shape[0], dev.ptr(t),
              dev.ptr(out), dev.stream_ptr())
    return out


def _gauss_prm(prm):
    return np.ascontiguousarray(prm, dtype=np.float64)


def prior_gauss(batch_size, seed, prm, offset=0):
    """Gaussian-model prior draws (elfi/examples/gauss.py:118-126): prm = [mu_lo, mu_width, a, b]."""
    mu, sigma = dev.empty((batch_size,)), dev.empty((batch_size,))
    _lib.call('elfi_b200_prior_gauss_f64', dev.context(), batch_size, int(seed), int(offset),
              dev.ptr(_gauss_prm(prm)), dev.ptr(mu), dev.ptr(sigma), dev.stream_ptr())
    return mu, sigma


def logprior_gauss(params, prm):
    x = _matrix(params)
    out = dev.empty((x.shape[0],))
    _lib.call('elfi_b200_logprior_gauss_f64', dev.context(), dev.ptr(x), _ld(x), x.shape[0],
              dev.ptr(_gauss_prm(prm)), dev.ptr(out), dev.stream_ptr())
    return out


def sim_gauss(mu, sigma, n_obs=50, seed=0, offset=0, want_data=False, want_summaries=True):
    """Gaussian simulator on the device -> (Y or None, S or None), S = [mean, var] fused."""
    mu = dev.to_device(mu).reshape(-1).contiguous()
    sigma = dev.to_device(sigma).reshape(-1).contiguous()
    B = mu.numel()
    Y = dev.empty((B, n_obs)) if want_data else None
    S = dev.empty((B, 2)) if want_summaries else None
    _lib.call('elfi_b200_sim_gauss_f64', dev.context(), dev.ptr(mu), dev.ptr(sigma), B, n_obs,
              int(seed), int(offset), dev.ptr(Y), n_obs, dev.ptr(S), 2, dev.stream_ptr())
    return Y, S


def sim_gnk(A, B, g, k, n_obs=50, seed=0, offset=0, c=0.8):
    """g-and-k simulator on the device (elfi/examples/gnk.py:11-68) -> Y (batch, n_obs)."""
    cols = [dev.to_device(v).reshape(-1).contiguous() for v in (A, B, g, k)]
    n = cols[0].numel()
    if any(col.numel() != n for col in cols):
        raise ValueError('A, B, g and k must have the same number of elements')
    Y = dev.empty((n, n_obs))
    _lib.call('elfi_b200_sim_gnk_f64', dev.context(), dev.ptr(cols[0]), dev.ptr(cols[1]),
              dev.ptr(cols[2]), dev.ptr(cols[3]), float(c), n, n_obs, int(seed), int(offset),
              dev.ptr(Y), n_obs, dev.stream_ptr())
    return Y


def logprior_box(params, lo, width):
    """Sum of independent uniform(lo, width) log densities per row (scipy convention: -inf
    outside); the joint prior of the g-and-k example (elfi/examples/gnk.py:99-103)."""
    x = _matrix(params)
    p = x.shape[1]
    box = np.ascontiguousarray(np.concatenate([np.broadcast_to(np.asarray(lo, dtype=np.float64), (p,)),
                                               np.broadcast_to(np.asarray(width, dtype=np.float64), (p,))]))
    out = dev.empty((x.shape[0],))
    _lib.call('elfi_b200_logprior_box_f64', dev.context(), dev.ptr(x), _ld(x), x.shape[0], p,
              dev.ptr(box), dev.ptr(out), dev.stream_ptr())
    return out


def kliep_fit(x, y, weights_x=None, weights_y=None, sigma=1.0, n_basis=100, epsilon=0.001,
              max_iter=200, abs_tol=0.01, conv_check_interval=20):
    """KLIEP fit on the device (elfi/methods/density_ratio_estimation.py:71-207).

    Returns (alpha device tensor (n_basis,), max_ratio float, steps int)."""
    x = _matrix(x)
    y = _matrix(y)
    if x.shape[0] < n_basis:
        raise ValueError("Number of RBFs ({}) can't be larger than number of samples ({}).".format(
            n_basis, x.shape[0]))
    wx = None if weights_x is None else dev.to_device(weights_x).reshape(-1)
    wy = None if weights_y is None else dev.to_device(weights_y).reshape(-1)
    alpha = dev.empty((n_basis,))
    res = (ctypes.c_double * 2)()
    dev.synchronize()   # this entry point runs on its own stream order: inputs must be complete
    _lib.call('elfi_b200_kliep_fit_f64', dev.context(), dev.ptr(x), _ld(x), x.shape[0], dev.ptr(y),
              _ld(y), y.shape[0], x.shape[1], dev.ptr(wx), dev.ptr(wy), float(sigma), int(n_basis),
              float(epsilon), int(max_iter), float(abs_tol), int(conv_check_interval),
              dev.ptr(alpha), res)
    return alpha, float(res[0]), int(res[1])


def rowsort(x):
    """np.sort(x, axis=1) on the device (ascending, NaN last); order-statistic summaries."""
    x = _matrix(x)
    B, n = x.shape
    out = dev.empty((B, n))
    _lib.call('elfi_b200_rowsort_f64', dev.context(), dev.ptr(x), _ld(x), B, n, dev.ptr(out), n,
              dev.stream_ptr())
    return out


# ---- robust / octile g-and-k summaries (elfi/examples/gnk.py:164-248, bignk.py) ------------------
GNK_KINDS = {'ss_robust': 0, 'ss_octile': 1}
GNK_WIDTH = {'ss_robust': 4, 'ss_octile': 7}
GNK_SERIES_MAX = _lib.CONSTANTS['GNK_SERIES_MAX']
GNK_FUSED_MAX = _lib.CONSTANTS['GNK_FUSED_MAX']
_GNK_OCTILES = np.linspace(12.5, 87.5, 7)


def gnk_picks(n):
    """Sorted positions and weights of np.percentile(y, [12.5, 25, .., 87.5], method='linear') for
    a series of length n, computed as numpy/lib/_function_base_impl.py does (_quantile,
    _get_indexes, _get_gamma): [lo (7), hi (7), t (7)] as a float64 array."""
    q = np.true_divide(_GNK_OCTILES, 100)
    vi = (n - 1) * q
    lo = np.floor(vi)
    hi = lo + 1
    above = vi >= n - 1
    lo[above] = -1
    hi[above] = -1
    t = vi - lo
    lo[lo < 0] = n - 1
    hi[hi < 0] = n - 1
    return np.ascontiguousarray(np.concatenate([lo, hi, t]), dtype=np.float64)


def _gnk_kind(kind):
    if kind not in GNK_KINDS:
        raise ValueError('unknown g-and-k summary {!r} (supported: {})'.format(
            kind, ', '.join(GNK_KINDS)))
    return GNK_KINDS[kind]


def gnk_summaries(y, kind='ss_robust'):
    """ss_robust / ss_octile of gnk.py on the device for y (B, n, d) (or (B, n) for d = 1),
    1 <= n <= 2048, d in {1, 2}: a (B, width * d) tensor laid out as the reference's np.hstack
    (reshape to (B, width * d, 1) for its shape), bit for bit."""
    k = _gnk_kind(kind)
    if not (dev.is_device_array(y) and y.dtype == torch.float64):
        y = dev.to_device(y)    # device views are read in place (row and observation strides)
    if y.dim() == 2:
        y = y[:, :, None]
    if y.dim() != 3:
        raise ValueError('expected (batch, n_obs, dim) data, got shape {}'.format(tuple(y.shape)))
    B, n, d = y.shape
    if d not in (1, 2):
        raise ValueError('g-and-k summaries take 1 or 2 dimensions, got {}'.format(d))
    if not 1 <= n <= GNK_SERIES_MAX:
        raise ValueError('g-and-k summaries on the device take 1 <= n_obs <= {}, got {}'.format(
            GNK_SERIES_MAX, n))
    if y.stride(2) != 1 or y.stride(1) < d:
        y = y.contiguous()
    out = dev.empty((B, GNK_WIDTH[kind] * d))
    _lib.call('elfi_b200_gnk_summaries_f64', dev.context(), dev.ptr(y),
              y.stride(0) if B > 1 else (n - 1) * y.stride(1) + d, y.stride(1), B, n, d, k,
              dev.ptr(gnk_picks(n)), dev.ptr(out), out.shape[1], dev.stream_ptr())
    return out


def sim_gnk_summaries(A, B, g, k, n_obs=50, seed=0, offset=0, c=0.8, kind='ss_robust'):
    """The ss_robust / ss_octile summaries of the rows :func:`sim_gnk` simulates for the same
    arguments, computed without writing the data: (batch, width), bit for bit equal to
    gnk_summaries(sim_gnk(...)).  n_obs <= 512."""
    kd = _gnk_kind(kind)
    if not 1 <= n_obs <= GNK_FUSED_MAX:
        raise ValueError('the fused g-and-k summaries take 1 <= n_obs <= {}, got {}'.format(
            GNK_FUSED_MAX, n_obs))
    cols = [dev.to_device(v).reshape(-1).contiguous() for v in (A, B, g, k)]
    n = cols[0].numel()
    if any(col.numel() != n for col in cols):
        raise ValueError('A, B, g and k must have the same number of elements')
    out = dev.empty((n, GNK_WIDTH[kind]))
    _lib.call('elfi_b200_sim_gnk_summaries_f64', dev.context(), dev.ptr(cols[0]), dev.ptr(cols[1]),
              dev.ptr(cols[2]), dev.ptr(cols[3]), float(c), n, int(n_obs), int(seed), int(offset), kd,
              dev.ptr(gnk_picks(n_obs)), dev.ptr(out), out.shape[1], dev.stream_ptr())
    return out


def sim_bignk(params, n_obs=150, seed=0, offset=0, c=0.8, want_data=True, kind=None):
    """Bivariate g-and-k simulator on the device (elfi/examples/bignk.py:12-108).  params: (batch, 9)
    columns A1, A2, B1, B2, g1, g2, k1, k2, rho.  Returns (Y (batch, n_obs, 2) or None,
    S (batch, 2 * width) or None): S = the fused ss_robust / ss_octile summaries when ``kind`` is
    given (n_obs <= 512), equal to gnk_summaries(Y, kind) bit for bit."""
    P = _matrix(params)
    if P.shape[1] != 9:
        raise ValueError('the bivariate g-and-k model has 9 parameters, got {}'.format(P.shape[1]))
    if n_obs < 1:
        raise ValueError('n_obs must be >= 1')
    kd, S = -1, None
    if kind is not None:
        kd = _gnk_kind(kind)
        if n_obs > GNK_FUSED_MAX:
            raise ValueError('the fused g-and-k summaries take n_obs <= {}, got {}'.format(
                GNK_FUSED_MAX, n_obs))
    B = P.shape[0]
    Y = dev.empty((B, n_obs, 2)) if want_data else None
    if kind is not None:
        S = dev.empty((B, 2 * GNK_WIDTH[kind]))
    _lib.call('elfi_b200_sim_bignk_f64', dev.context(), dev.ptr(P), _ld(P), float(c), B,
              int(n_obs), int(seed), int(offset), dev.ptr(Y), 2 * n_obs, kd,
              dev.ptr(gnk_picks(n_obs)) if kind is not None else None, dev.ptr(S),
              S.shape[1] if S is not None else 0, dev.stream_ptr())
    return Y, S


def euclidean_multiss(S, obs):
    """euclidean_multiss of gnk.py:115-142 for device summaries S (B, K) or (B, K, 1) and observed
    summaries obs (K,) / (1, K, 1), K <= 128: sqrt(sum_j (S[:, j] - obs[j])^2) in NumPy's order,
    bit for bit.  Returns a device tensor (B,)."""
    if dev.is_device_array(S) and S.dim() == 3:
        if S.shape[2] != 1:
            raise ValueError('euclidean_multiss on the device takes (B, K, 1) summaries')
        S = S[:, :, 0]
    S = _matrix(S)
    B, K = S.shape
    o = np.ascontiguousarray(np.asarray(dev.to_host(obs) if dev.is_device_array(obs) else obs,
                                        dtype=np.float64).reshape(-1))
    if o.size != K:
        raise ValueError('observed summaries have {} values, simulated {}'.format(o.size, K))
    if not 1 <= K <= 128:
        raise ValueError('euclidean_multiss on the device takes 1 <= K <= 128 summaries, got {}'
                         .format(K))
    o = dev.to_device(o)
    out = dev.empty((B,))
    _lib.call('elfi_b200_euclidean_multiss_f64', dev.context(), dev.ptr(S), _ld(S), B, K,
              dev.ptr(o), dev.ptr(out), dev.stream_ptr())
    return out


# ---- Ricker model (elfi/examples/ricker.py) -------------------------------------------------------
POISSON_LAM_MAX = _lib.CONSTANTS['POISSON_LAM_MAX']
RICKER_FUSED_MAX = _lib.CONSTANTS['RICKER_FUSED_MAX']
RICKER_NOBS_MAX = _lib.CONSTANTS['RICKER_NOBS_MAX']


def poisson(lam, seed, offset=0):
    """Poisson(lam) draws on the device, one per element of lam (any shape): element i (in C order)
    is a pure function of (seed, offset + i).  lam == 0 gives 0; lam < 0, NaN or lam >
    POISSON_LAM_MAX give NaN (where NumPy raises).  Returns float64 counts shaped like lam."""
    lam = dev.to_device(lam)
    flat = lam.reshape(-1).contiguous()
    out = dev.empty((flat.numel(),))
    _lib.call('elfi_b200_poisson_f64', dev.context(), dev.ptr(flat), flat.numel(), int(seed),
              int(offset), dev.ptr(out), dev.stream_ptr())
    return out.reshape(lam.shape)


def _ricker_params(params, stochastic):
    P = _matrix(params)
    p = 3 if stochastic else 1
    if P.shape[1] != p:
        raise ValueError('the {} Ricker model has {} parameter{}, got {}'.format(
            'stochastic' if stochastic else 'deterministic', p, 's' if p > 1 else '', P.shape[1]))
    return P


def sim_ricker(params, n_obs=50, seed=0, offset=0, stochastic=True, stock_init=1.0, want_data=False,
               want_latent=False, want_summaries=True):
    """Ricker simulator on the device (elfi/examples/ricker.py:11-85).  params: (batch, 3) columns
    log_rate, std, scale for the stochastic model, (batch, 1) or (batch,) log_rate for the
    deterministic one.  Row i is a pure function of (seed, offset + i).

    Returns (Y, N, S), each None unless asked for: Y (batch, n_obs) the observed counts (the stock
    for the deterministic model), N (batch, n_obs) the latent stock, S (batch, 3) =
    [np.mean(Y), np.var(Y), number of zeros of Y] per row.  For n_obs <= RICKER_FUSED_MAX S is
    computed in the simulator without writing Y; above, Y is written and summarised
    (:func:`ricker_summaries`).  Both give the same bits."""
    if np.ndim(stock_init) != 0:
        raise ValueError('stock_init must be a scalar on the device, got shape {}'.format(
            np.shape(stock_init)))
    if not 1 <= int(n_obs) <= RICKER_NOBS_MAX:
        raise ValueError('the device Ricker simulator takes 1 <= n_obs <= {}, got {}'.format(
            RICKER_NOBS_MAX, n_obs))
    n_obs = int(n_obs)
    P = _ricker_params(params, stochastic)
    B = P.shape[0]
    fused = want_summaries and n_obs <= RICKER_FUSED_MAX
    Y = dev.empty((B, n_obs)) if want_data or (want_summaries and not fused) else None
    N = dev.empty((B, n_obs)) if want_latent else None
    S = dev.empty((B, 3)) if fused else None
    _lib.call('elfi_b200_sim_ricker_f64', dev.context(), dev.ptr(P), _ld(P), P.shape[1], B, n_obs,
              float(stock_init), int(seed), int(offset), dev.ptr(Y), n_obs, dev.ptr(N), n_obs,
              dev.ptr(S), 3, dev.stream_ptr())
    if want_summaries and not fused:
        S = ricker_summaries(Y)
    return (Y if want_data else None), N, S


def count_zeros(y, out=None):
    """num_zeros of elfi/examples/ricker.py:164-167 on the device: the number of zeros of each row
    of y (B, n), as float64 (B,) (or into the column view ``out``)."""
    y = _matrix(y)
    B, n = y.shape
    out = _out(out, (B,), 'count_zeros')
    _lib.call('elfi_b200_count_zeros_f64', dev.context(), dev.ptr(y), _ld(y), B, n, dev.ptr(out),
              out.stride(0) if B > 1 else 1, dev.stream_ptr())
    return out


def ricker_summaries(y):
    """The Ricker summaries [np.mean, np.var, num_zeros] of each row of device data y (B, n): a
    (B, 3) tensor, bit for bit NumPy's (mean and variance from :func:`meanvar`)."""
    y = _matrix(y)
    S = dev.empty((y.shape[0], 3))
    meanvar(y, out=S[:, :2])
    count_zeros(y, out=S[:, 2])
    return S


def chi_squared(S, obs):
    """chi_squared of elfi/examples/ricker.py:147-161 for device summaries S (B, K) and observed
    summaries obs (K,), K <= 128: sum_j (S[:, j] - obs[j])^2 / obs[j] in NumPy's order, bit for
    bit (obs[j] = 0 gives NumPy's inf / NaN).  Returns a device tensor (B,)."""
    S = _matrix(S)
    B, K = S.shape
    o = np.ascontiguousarray(np.asarray(dev.to_host(obs) if dev.is_device_array(obs) else obs,
                                        dtype=np.float64).reshape(-1))
    if o.size != K:
        raise ValueError('observed summaries have {} values, simulated {}'.format(o.size, K))
    if not 1 <= K <= 128:
        raise ValueError('chi_squared on the device takes 1 <= K <= 128 summaries, got {}'.format(K))
    o = dev.to_device(o)
    out = dev.empty((B,))
    _lib.call('elfi_b200_chi_squared_f64', dev.context(), dev.ptr(S), _ld(S), B, K, dev.ptr(o),
              dev.ptr(out), dev.stream_ptr())
    return out


RICKER_WOOD_NOBS_MIN = _lib.CONSTANTS['RICKER_WOOD_NOBS_MIN']
RICKER_WOOD_NOBS_MAX = _lib.CONSTANTS['RICKER_WOOD_NOBS_MAX']
RICKER_WOOD_WIDTH = _lib.CONSTANTS['RICKER_WOOD_WIDTH']


def wood_summaries(y, design):
    """Wood's 13 Ricker statistics (ss_wood of elfi_b200.examples.ricker) of each row of y (B, n),
    7 <= n <= RICKER_WOOD_NOBS_MAX, on the device.  design: the (3, n - 1) pseudo-inverse of the
    observed series' cubic design (ricker.wood_design), a host array or, to avoid a copy per call,
    a device tensor.  Returns a (B, 13) device tensor; accuracy in include/elfi_b200.h."""
    y = _matrix(y)
    B, n = y.shape
    if not RICKER_WOOD_NOBS_MIN <= n <= RICKER_WOOD_NOBS_MAX:
        raise ValueError("Wood's statistics on the device take {} <= n_obs <= {}, got {}".format(
            RICKER_WOOD_NOBS_MIN, RICKER_WOOD_NOBS_MAX, n))
    if tuple(design.shape) != (3, n - 1):
        raise ValueError('the cubic design of a series of {} values is (3, {}), got shape {}'.format(
            n, n - 1, tuple(design.shape)))
    P = dev.to_device(design)
    out = dev.empty((B, RICKER_WOOD_WIDTH))
    _lib.call('elfi_b200_ricker_wood_f64', dev.context(), dev.ptr(y), _ld(y), B, n, dev.ptr(P),
              dev.ptr(out), RICKER_WOOD_WIDTH, dev.stream_ptr())
    return out


# ---- Lorenz forecast model (elfi/examples/lorenz.py) ----------------------------------------------
LORENZ_NOBS_MIN = _lib.CONSTANTS['LORENZ_NOBS_MIN']
LORENZ_NOBS_MAX = _lib.CONSTANTS['LORENZ_NOBS_MAX']
LORENZ_SUMM_NOBS_MIN = _lib.CONSTANTS['LORENZ_SUMM_NOBS_MIN']
LORENZ_T_MAX = _lib.CONSTANTS['LORENZ_T_MAX']
LORENZ_SUMM_MAX_TERMS = _lib.CONSTANTS['LORENZ_SUMM_MAX_TERMS']
LORENZ_NSUMM = 6


def sim_lorenz(params, n_timestep=160, initial_state=None, f=10., phi=0.984, total_duration=4.,
               seed=0, offset=0, want_data=False, want_summaries=True):
    """Stochastic Lorenz 96 forecast model on the device (elfi/examples/lorenz.py:94-163).
    params: (batch, 2) columns theta1, theta2.  initial_state: the n_obs values of time 0 (default:
    the reference's 40-value state, examples.lorenz.INITIAL_STATE); 4 <= n_obs <= 128.  Row i is a
    pure function of (seed, offset + i).  dt = total_duration / n_timestep and
    sqrt(1 - phi ** 2) are computed as the reference computes them (phi > 1 gives NaN rows).

    Returns (X, S), each None unless asked for: X (batch, n_timestep, n_obs) the trajectories, S
    (batch, 6) = [Mean, Var, Autocov, Cov, CrosscovPrev, CrosscovNext] per row.  Without want_data
    the summaries are computed in the simulator and no (batch, n_timestep, n_obs) tensor is
    allocated; either way S equals :func:`lorenz_summaries` of X bit for bit."""
    if initial_state is None:
        from .examples.lorenz import INITIAL_STATE
        initial_state = INITIAL_STATE
    init = np.array(initial_state, dtype=np.float64)      # a writable copy for torch
    if init.ndim != 1:
        raise ValueError('initial_state must be one vector of n_obs values, got shape {}'.format(
            init.shape))
    m = init.size
    if not LORENZ_NOBS_MIN <= m <= LORENZ_NOBS_MAX:
        raise ValueError('the device Lorenz simulator takes an initial state of {} <= n_obs <= {} '
                         'values, got {}'.format(LORENZ_NOBS_MIN, LORENZ_NOBS_MAX, m))
    n_timestep = int(n_timestep)
    if not 2 <= n_timestep <= LORENZ_T_MAX:
        raise ValueError('the device Lorenz simulator takes 2 <= n_timestep <= {}, got {}'.format(
            LORENZ_T_MAX, n_timestep))
    if want_summaries and n_timestep * m > LORENZ_SUMM_MAX_TERMS:
        raise ValueError('the device Lorenz summaries take n_timestep * n_obs <= {}, got {} * {}'
                         .format(LORENZ_SUMM_MAX_TERMS, n_timestep, m))
    P = _params(params, 'Lorenz', ('theta1', 'theta2'))
    B = P.shape[0]
    dt = total_duration / n_timestep
    with np.errstate(invalid='ignore'):
        s_phi = float(np.sqrt(1 - pow(phi, 2)))
    X = dev.empty((B, n_timestep, m)) if want_data else None
    S = dev.empty((B, LORENZ_NSUMM)) if want_summaries else None
    _lib.call('elfi_b200_sim_lorenz_f64', dev.context(), dev.ptr(P), _ld(P), B, m, n_timestep,
              dev.ptr(dev.to_device(init)), float(f), float(phi), s_phi, float(dt), int(seed),
              int(offset), dev.ptr(X), dev.ptr(S), LORENZ_NSUMM, dev.stream_ptr())
    return X, S


def lorenz_summaries(x):
    """The six Lorenz summaries [Mean, Var, Autocov, Cov, CrosscovPrev, CrosscovNext]
    (elfi/examples/lorenz.py:231-320) of device data x (B, n_timestep, n_obs), any strides: a
    (B, 6) tensor, bit for bit NumPy's on the C-contiguous array.  2 <= n_timestep,
    2 <= n_obs <= 128, n_timestep * n_obs <= LORENZ_SUMM_MAX_TERMS."""
    x = _data(x, 'lorenz_summaries', ('batch', 'n_timestep', 'n_obs'))
    B, T, m = x.shape
    if not LORENZ_SUMM_NOBS_MIN <= m <= LORENZ_NOBS_MAX or T < 2 or T * m > LORENZ_SUMM_MAX_TERMS:
        raise ValueError('lorenz_summaries takes {} <= n_obs <= {}, 2 <= n_timestep and n_timestep * '
                         'n_obs <= {}, got n_timestep {}, n_obs {}'.format(
                             LORENZ_SUMM_NOBS_MIN, LORENZ_NOBS_MAX, LORENZ_SUMM_MAX_TERMS, T, m))
    S = dev.empty((B, LORENZ_NSUMM))
    _lib.call('elfi_b200_lorenz_summaries_f64', dev.context(), dev.ptr(x), x.stride(0), x.stride(1),
              x.stride(2), B, T, m, dev.ptr(S), LORENZ_NSUMM, dev.stream_ptr())
    return S


# ---- Toad movement model (elfi/examples/toad.py) --------------------------------------------------
TOAD_DISP_MAX = _lib.CONSTANTS['TOAD_DISP_MAX']
TOAD_LAGS_MAX = _lib.CONSTANTS['TOAD_LAGS_MAX']
TOAD_NP_MAX = _lib.CONSTANTS['TOAD_NP_MAX']
TOAD_CELLS_MAX = _lib.CONSTANTS['TOAD_CELLS_MAX']


def _toad_p(p):
    p = np.array(p, dtype=np.float64).reshape(-1)
    if not 1 <= p.size <= TOAD_NP_MAX:
        raise ValueError('the toad summaries take 1 <= len(p) <= {} quantile levels, got {}'.format(
            TOAD_NP_MAX, p.size))
    if not np.all((p >= 0) & (p <= 1)):
        raise ValueError('the toad quantile levels p must lie in [0, 1]')
    return np.ascontiguousarray(p)


def _toad_lag(lag, n_days):
    if int(lag) != lag or not 1 <= lag < n_days:
        raise ValueError('the toad summaries take an integer lag with 1 <= lag < n_days = {}, got {}'
                         .format(n_days, lag))
    return int(lag)


def _toad_disp(n_toads, rows):
    if n_toads * rows > TOAD_DISP_MAX:
        raise ValueError('the device toad summaries take n_toads * (n_days - lag) <= {} '
                         'displacements, got {} * {}'.format(TOAD_DISP_MAX, n_toads, rows))


def sim_toad(params, n_toads=66, n_days=63, seed=0, offset=0, want_data=False, lags=(1, 2, 4, 8),
             p=np.linspace(0, 1, 11), thd=10.):
    """Toad movement simulator on the device (elfi/examples/toad.py:16-70).  params: (batch, 3)
    columns alpha, gamma, p0.  Row i is a pure function of (seed, offset + i); alpha outside (0, 2]
    or gamma < 0 (where the reference raises) give rows of NaN.

    Returns (X, S), each None unless asked for: X (batch, n_days, n_toads) the positions (batch
    first; ``X.permute(1, 2, 0)`` is indexed like the reference's array), S (batch, len(lags) *
    (len(p) + 1)) the summaries of each lag (:func:`toad_summaries`) side by side; lags=None or ()
    asks for no summaries.  Without want_data the summaries are computed in the simulator and no
    (batch, n_days, n_toads) tensor is allocated; either way S equals :func:`toad_summaries` of X bit
    for bit.  Limits: n_days * n_toads <= TOAD_CELLS_MAX; for the summaries n_toads * (n_days - 1)
    <= TOAD_DISP_MAX, at most TOAD_LAGS_MAX lags and TOAD_NP_MAX levels."""
    n_toads, n_days = int(n_toads), int(n_days)
    if n_toads < 1 or n_days < 1 or n_toads * n_days > TOAD_CELLS_MAX:
        raise ValueError('the device toad simulator takes n_toads >= 1, n_days >= 1 and '
                         'n_days * n_toads <= {}, got {} * {}'.format(TOAD_CELLS_MAX, n_days,
                                                                      n_toads))
    lags = () if lags is None else tuple(lags)
    if len(lags) > TOAD_LAGS_MAX:
        raise ValueError('the device toad simulator fuses at most {} lags, got {}'.format(
            TOAD_LAGS_MAX, len(lags)))
    lag_arr = pv = None
    if lags:
        lag_arr = np.array([_toad_lag(lag, n_days) for lag in lags], dtype=np.int64)
        _toad_disp(n_toads, n_days - 1)
        pv = _toad_p(p)
    P = _params(params, 'toad', ('alpha', 'gamma', 'p0'))
    B = P.shape[0]
    X = dev.empty((B, n_days, n_toads)) if want_data else None
    w = len(lags) * (pv.size + 1) if lags else 0
    S = dev.empty((B, w)) if lags else None
    _lib.call('elfi_b200_sim_toad_f64', dev.context(), dev.ptr(P), _ld(P), B, n_toads, n_days,
              int(seed), int(offset), dev.ptr(X), len(lags), dev.ptr(lag_arr),
              0 if pv is None else pv.size, dev.ptr(pv), float(thd), dev.ptr(S), w, dev.stream_ptr())
    return X, S


def toad_summaries(x, lag, p=np.linspace(0, 1, 11), thd=10.):
    """compute_summaries of elfi/examples/toad.py:73-132 for device data x (n_days, n_toads, batch),
    any strides: a (batch, len(p) + 1) tensor [number of returns, median, len(p) - 1 log gaps], bit
    for bit NumPy's except that the logs use the device's log.  1 <= lag < n_days, n_toads *
    (n_days - lag) <= TOAD_DISP_MAX, 1 <= len(p) <= TOAD_NP_MAX levels in [0, 1]."""
    x = _data(x, 'toad_summaries', ('n_days', 'n_toads', 'batch'))
    n_days, n_toads, B = x.shape
    lag = _toad_lag(lag, n_days)
    _toad_disp(n_toads, n_days - lag)
    pv = _toad_p(p)
    S = dev.empty((B, pv.size + 1))
    _lib.call('elfi_b200_toad_summaries_f64', dev.context(), dev.ptr(x), x.stride(0), x.stride(1),
              x.stride(2), n_days, n_toads, B, lag, pv.size, dev.ptr(pv), float(thd), dev.ptr(S),
              pv.size + 1, dev.stream_ptr())
    return S


# ---- Lotka-Volterra model (elfi/examples/lotka_volterra.py) ----------------------------------------
LV_NOBS_MAX = _lib.CONSTANTS['LV_NOBS_MAX']
LV_SUMM_NOBS_MIN = _lib.CONSTANTS['LV_SUMM_NOBS_MIN']
LV_SUMM_NOBS_MAX = _lib.CONSTANTS['LV_SUMM_NOBS_MAX']
LV_NSUMM = _lib.CONSTANTS['LV_NSUMM']
LV_MAX_EVENTS_LIMIT = _lib.CONSTANTS['LV_MAX_EVENTS_LIMIT']


def sim_lotka_volterra(params, n_obs=16, time_end=30., seed=0, offset=0, max_events=2 ** 20):
    """Lotka-Volterra simulator on the device (elfi/examples/lotka_volterra.py:18-143), Gillespie's
    direct method per row.  params: (batch, 6) columns r1, r2, r3, prey0, predator0, sigma.  Row i is
    a pure function of (seed, offset + i).

    Returns (obs, n_events): obs (batch, n_obs, 2) float64 holding the int32 counts of prey and
    predators at np.linspace(0, time_end, n_obs) (with noise sigma), n_events (batch,) int64 the
    events each row ran.  A row that has not reached time_end after max_events events, or whose
    parameters the reference rejects (a negative or NaN rate or sigma, floor(prey0) or
    floor(predator0) outside [0, 2^31)), gets NaN observations; a capped row reports
    n_events == max_events.  1 <= n_obs <= LV_NOBS_MAX, time_end finite and > 0,
    1 <= max_events <= LV_MAX_EVENTS_LIMIT."""
    n_obs = int(n_obs)
    if not 1 <= n_obs <= LV_NOBS_MAX:
        raise ValueError('the device Lotka-Volterra simulator takes 1 <= n_obs <= {}, got {}'.format(
            LV_NOBS_MAX, n_obs))
    time_end = float(time_end)
    if not (np.isfinite(time_end) and time_end > 0):
        raise ValueError('the device Lotka-Volterra simulator takes a finite time_end > 0, got '
                         '{}'.format(time_end))
    if int(max_events) != max_events or not 1 <= max_events <= LV_MAX_EVENTS_LIMIT:
        raise ValueError('max_events must be an integer with 1 <= max_events <= {} (the event '
                         'index is one Philox word), got {}'.format(LV_MAX_EVENTS_LIMIT, max_events))
    P = _params(params, 'Lotka-Volterra', ('r1', 'r2', 'r3', 'prey0', 'predator0', 'sigma'))
    B = P.shape[0]
    t_out = dev.to_device(np.linspace(0, time_end, n_obs))
    obs = dev.empty((B, n_obs, 2))
    n_events = dev.empty((B,), dtype=torch.int64)
    _lib.call('elfi_b200_sim_lotka_volterra_f64', dev.context(), dev.ptr(P), _ld(P), B,
              dev.ptr(t_out), n_obs, time_end, int(max_events), int(seed), int(offset),
              dev.ptr(obs), dev.ptr(n_events), dev.stream_ptr())
    return obs, n_events


def lv_summaries(x):
    """The nine summaries of elfi/examples/lotka_volterra.py:206-277 for device data x
    (batch, n_obs, 2), any strides: a (batch, 9) tensor [prey_mean, pred_mean, prey_log_var,
    pred_log_var, prey_autocorr_1, pred_autocorr_1, prey_autocorr_2, pred_autocorr_2, crosscorr],
    bit for bit NumPy's except that log(var + 1) uses the device's log.
    LV_SUMM_NOBS_MIN <= n_obs <= LV_SUMM_NOBS_MAX."""
    x = _data(x, 'lv_summaries', ('batch', 'n_obs', 2))
    B, n_obs = x.shape[0], x.shape[1]
    if not LV_SUMM_NOBS_MIN <= n_obs <= LV_SUMM_NOBS_MAX:
        raise ValueError('the device Lotka-Volterra summaries take {} <= n_obs <= {}, got {}'.format(
            LV_SUMM_NOBS_MIN, LV_SUMM_NOBS_MAX, n_obs))
    S = dev.empty((B, LV_NSUMM))
    _lib.call('elfi_b200_lv_summaries_f64', dev.context(), dev.ptr(x), x.stride(0), x.stride(1),
              x.stride(2), B, n_obs, dev.ptr(S), LV_NSUMM, dev.stream_ptr())
    return S


# ---- birth-death-mutation model (elfi/examples/bdm.py) ----------------------------------------
BDM_N_MAX = _lib.CONSTANTS['BDM_N_MAX']
BDM_NSUMM = _lib.CONSTANTS['BDM_NSUMM']
BDM_MAX_EVENTS_LIMIT = _lib.CONSTANTS['BDM_MAX_EVENTS_LIMIT']
BDM_BATCH_MAX = _lib.CONSTANTS['BDM_BATCH_MAX']


def _bdm_N(N):
    if int(N) != N or not 1 <= N <= BDM_N_MAX:
        raise ValueError('the device BDM model takes an integer 1 <= N <= {}, got {}'.format(
            BDM_N_MAX, N))
    return int(N)


def sim_bdm(params, N, seed=0, offset=0, max_events=2 ** 24, n=20, want_data=True,
            want_summaries=True):
    """Birth-death-mutation simulator on the device: the law of the reference's executable
    elfi/examples/cpp/bdm.cpp with --mode 1.  params: (batch, 3) columns alpha (birth), delta
    (death), tau (mutation).  Row i is a pure function of (seed, offset + i).

    Returns (X, S, n_events): X (batch, N) int16 cluster sizes (None unless want_data), S (batch, 2)
    the summaries T1 and T2 with T2's argument n (None unless want_summaries), bit for bit
    :func:`bdm_summaries` of X, and n_events (batch,) int64 the events each row ran.  A row with a
    rate that is negative, NaN or infinite, or with a total rate of 0, gets counts of -1, NaN
    summaries and n_events = -1; a row still running after max_events events gets counts of -1,
    NaN summaries and n_events = max_events.  1 <= N <= BDM_N_MAX,
    1 <= max_events <= BDM_MAX_EVENTS_LIMIT, batch < 2^31."""
    N = _bdm_N(N)
    if int(max_events) != max_events or not 1 <= max_events <= BDM_MAX_EVENTS_LIMIT:
        raise ValueError('max_events must be an integer with 1 <= max_events <= {} (the event '
                         'index is one Philox word), got {}'.format(BDM_MAX_EVENTS_LIMIT,
                                                                    max_events))
    P = _params(params, 'BDM', ('alpha', 'delta', 'tau'))
    B = P.shape[0]
    if B > BDM_BATCH_MAX:
        raise ValueError('the device BDM simulator takes at most {} rows per call, got {}'.format(
            BDM_BATCH_MAX, B))
    X = dev.empty((B, N), dtype=torch.int16) if want_data else None
    S = dev.empty((B, BDM_NSUMM)) if want_summaries else None
    n_events = dev.empty((B,), dtype=torch.int64)
    _lib.call('elfi_b200_sim_bdm_f64', dev.context(), dev.ptr(P), _ld(P), B, N, float(n),
              int(max_events), int(seed), int(offset), dev.ptr(X), N, dev.ptr(S), BDM_NSUMM,
              dev.ptr(n_events), dev.stream_ptr())
    return X, S, n_events


def bdm_summaries(x, n=20):
    """T1 and T2 of elfi/examples/bdm.py for device cluster sizes x (batch, N), any strides: a
    (batch, 2) tensor, bit for bit NumPy's T1(x) and T2(x, n) and :func:`sim_bdm`'s.  int16
    device data is read in place; anything else is cast to int16 (host data is uploaded first).
    A row with a negative count (the mark of sim_bdm's invalid and capped rows) gets NaN.
    1 <= N <= BDM_N_MAX."""
    if not dev.is_device_array(x):
        x = dev.to_device(torch.from_numpy(np.ascontiguousarray(x, dtype=np.int16)),
                          dtype=torch.int16)
    if x.dtype != torch.int16:
        x = x.to(torch.int16)
    if x.dim() == 1:
        x = x[None, :]
    _axes(x, 'bdm_summaries', ('batch', 'N'))
    B, N = int(x.shape[0]), _bdm_N(int(x.shape[1]))
    S = dev.empty((B, BDM_NSUMM))
    _lib.call('elfi_b200_bdm_summaries_f64', dev.context(), dev.ptr(x), x.stride(0), x.stride(1),
              B, N, float(n), dev.ptr(S), BDM_NSUMM, dev.stream_ptr())
    return S


# ---- day care model (elfi/examples/daycare.py) ----------------------------------------------------
DC_DCC_MAX = _lib.CONSTANTS['DC_DCC_MAX']
DC_IND_MAX = _lib.CONSTANTS['DC_IND_MAX']
DC_STRAINS_MAX = _lib.CONSTANTS['DC_STRAINS_MAX']
DC_SUMM_STRAINS_MAX = _lib.CONSTANTS['DC_SUMM_STRAINS_MAX']
DC_NSUMM = _lib.CONSTANTS['DC_NSUMM']
DC_DIST_TERMS_MAX = _lib.CONSTANTS['DC_DIST_TERMS_MAX']
DC_BATCH_MAX = _lib.CONSTANTS['DC_BATCH_MAX']


def sim_daycare(params, n_dcc=29, n_ind=53, n_strains=33, freq_strains_commun=None, n_obs=36,
                time_end=10., seed=0, offset=0, want_data=False, want_summaries=True):
    """Day care simulator on the device (elfi/examples/daycare.py:16-141), Gillespie's direct
    method in each DCC.  params: (batch, 3) columns t1, t2, t3.  Within a row every DCC takes as
    many transitions as the DCC that needs most to pass time_end (the reference's law at
    batch_size=1); row i is a pure function of (seed, offset + i).

    Returns (summaries, data, K): summaries (batch, 4 n_dcc) float64 in column blocks
    [Shannon | n_strains | prevalence | multi] of the first n_obs children (None unless
    want_summaries), data (batch, n_dcc, n_obs, n_strains) bool (None unless want_data), K (batch,)
    int64 the transitions each row took.  A row whose t1, t2 or t3 is negative, NaN or infinite, or
    whose expected transitions per DCC could reach 2^32 - 1 (time_end n_ind n_strains
    max(1, max(1, t3) (t1 + 1e-9 + t2 max(freq_strains_commun))) >= 2^32 - 1), gets NaN summaries,
    all-False data and K = -1.  Limits: n_dcc <= DC_DCC_MAX, 2 <= n_ind <= DC_IND_MAX,
    n_strains <= DC_STRAINS_MAX, 1 <= n_obs <= n_ind, freq_strains_commun finite and >= 0,
    time_end finite and > 0."""
    n_dcc, n_ind, n_strains, n_obs = int(n_dcc), int(n_ind), int(n_strains), int(n_obs)
    if not (1 <= n_dcc <= DC_DCC_MAX and 2 <= n_ind <= DC_IND_MAX
            and 1 <= n_strains <= DC_STRAINS_MAX):
        raise ValueError('the device day care simulator takes 1 <= n_dcc <= {}, 2 <= n_ind <= {} '
                         'and 1 <= n_strains <= {}, got n_dcc={}, n_ind={}, n_strains={}'.format(
                             DC_DCC_MAX, DC_IND_MAX, DC_STRAINS_MAX, n_dcc, n_ind, n_strains))
    if not 1 <= n_obs <= n_ind:
        raise ValueError('the device day care simulator takes 1 <= n_obs <= n_ind, got n_obs={}, '
                         'n_ind={}'.format(n_obs, n_ind))
    time_end = float(time_end)
    if not (np.isfinite(time_end) and time_end > 0):
        raise ValueError('the device day care simulator takes a finite time_end > 0, got '
                         '{}'.format(time_end))
    if freq_strains_commun is None:
        freq_strains_commun = np.full(n_strains, 0.1)
    f = np.asarray(dev.to_host(freq_strains_commun), dtype=np.float64).reshape(-1)
    if f.size != n_strains:
        raise ValueError('freq_strains_commun must have n_strains = {} values, got {}'.format(
            n_strains, f.size))
    if not (np.all(np.isfinite(f)) and np.all(f >= 0)):
        raise ValueError('freq_strains_commun must be finite and >= 0, got {}'.format(f))
    P = _params(params, 'day care', ('t1', 't2', 't3'))
    B = P.shape[0]
    if B > DC_BATCH_MAX:
        raise ValueError('the device day care simulator takes at most {} rows per call, got '
                         '{}'.format(DC_BATCH_MAX, B))
    S = dev.empty((B, DC_NSUMM * n_dcc)) if want_summaries else None
    X = dev.empty((B, n_dcc, n_obs, n_strains), dtype=torch.bool) if want_data else None
    K = dev.empty((B,), dtype=torch.int64)
    fd = dev.to_device(f)
    _lib.call('elfi_b200_sim_daycare_f64', dev.context(), dev.ptr(P), _ld(P), B, n_dcc, n_ind,
              n_strains, dev.ptr(fd), n_obs, time_end, int(seed), int(offset), dev.ptr(S),
              DC_NSUMM * n_dcc, dev.ptr(X), dev.ptr(K), dev.stream_ptr())
    return S, X, K


def daycare_summaries(data):
    """The four summaries of elfi/examples/daycare.py:199-275 for device data (batch, n_dcc, n_obs,
    n_strains), any strides, nonzero meaning a carrier: a (batch, 4 n_dcc) tensor in column blocks
    [Shannon | n_strains | prevalence | multi], bit for bit NumPy's except that Shannon uses the
    device's log.  n_strains <= DC_SUMM_STRAINS_MAX."""
    data = _mask(data, 'daycare_summaries', ('batch', 'n_dcc', 'n_obs', 'n_strains'))
    B, n_dcc, n_obs, n_strains = (int(v) for v in data.shape)
    if n_dcc < 1 or n_obs < 1 or not 1 <= n_strains <= DC_SUMM_STRAINS_MAX:
        raise ValueError('the device day care summaries take n_dcc, n_obs >= 1 and 1 <= n_strains '
                         '<= {}, got shape {}'.format(DC_SUMM_STRAINS_MAX, tuple(data.shape)))
    S = dev.empty((B, DC_NSUMM * n_dcc))
    _lib.call('elfi_b200_daycare_summaries_f64', dev.context(), dev.ptr(data), data.stride(0),
              data.stride(1), data.stride(2), data.stride(3), B, n_dcc, n_obs, n_strains,
              dev.ptr(S), DC_NSUMM * n_dcc, dev.stream_ptr())
    return S


def daycare_observed(observed):
    """The observed side of daycare_distance from the k (1, n_dcc) observed summaries, on the host:
    (obs_max (k,), y (k, n_dcc)) with obs_max the per-summary maximum (0 replaced by 1) and y the
    observed values divided by it and sorted (elfi/examples/daycare.py:296-306)."""
    observed = np.stack([np.asarray(dev.to_host(o), dtype=np.float64) for o in observed])
    obs_max = np.max(observed, axis=2, keepdims=True)
    obs_max = np.where(obs_max == 0, 1, obs_max)
    y = np.sort(observed / obs_max, axis=2)
    return obs_max.reshape(-1), y.reshape(len(observed), -1)


def daycare_distance(S, observed, n_dcc):
    """The distance of elfi/examples/daycare.py:278-312 on the device: S (batch, k n_dcc) holds the
    k simulated summaries side by side, observed the k (1, n_dcc) observed ones.  Each row is
    divided by the observed maxima, sorted per summary (NaN last), and its mean absolute difference
    from the sorted observed values is taken, bit for bit as NumPy does (one pairwise sum for a
    batch of one row, else one per summary, added in order).  k n_dcc <= DC_DIST_TERMS_MAX."""
    S = _matrix(S)
    n_dcc = int(n_dcc)
    k = len(observed)
    if S.shape[1] != k * n_dcc or not 1 <= k * n_dcc <= DC_DIST_TERMS_MAX:
        raise ValueError('daycare_distance takes {} summaries of n_dcc = {} columns, at most {} '
                         'values per row; got a width of {}'.format(k, n_dcc, DC_DIST_TERMS_MAX,
                                                                    S.shape[1]))
    obs_max, y = daycare_observed(observed)
    if y.shape[1] != n_dcc:
        raise ValueError('the observed summaries have {} DCCs, the simulated ones {}'.format(
            y.shape[1], n_dcc))
    om, yd = dev.to_device(obs_max), dev.to_device(y)
    B = S.shape[0]
    d = dev.empty((B,))
    _lib.call('elfi_b200_daycare_distance_f64', dev.context(), dev.ptr(S), _ld(S), B, k, n_dcc,
              dev.ptr(om), dev.ptr(yd), dev.ptr(d), dev.stream_ptr())
    return d


# ---- ARCH(1) model (elfi/examples/arch.py) --------------------------------------------------------
ARCH_NOBS_MIN = _lib.CONSTANTS['ARCH_NOBS_MIN']
ARCH_NOBS_MAX = _lib.CONSTANTS['ARCH_NOBS_MAX']
ARCH_LAGS_MAX = _lib.CONSTANTS['ARCH_LAGS_MAX']


def arch_nsumm(n_lags):
    """The number of ARCH summaries for n_lags lags: MU, VAR, the n_lags AC and their pairwise
    products."""
    return 2 + n_lags + n_lags * (n_lags - 1) // 2


def _arch_shape(n_obs, n_lags, what):
    if int(n_obs) != n_obs or not ARCH_NOBS_MIN <= n_obs <= ARCH_NOBS_MAX:
        raise ValueError('{} take {} <= n_obs <= {}, got {}'.format(what, ARCH_NOBS_MIN,
                                                                    ARCH_NOBS_MAX, n_obs))
    top = min(ARCH_LAGS_MAX, int(n_obs) - 1)
    if int(n_lags) != n_lags or not 1 <= n_lags <= top:
        raise ValueError('{} take 1 <= n_lags <= min({}, n_obs - 1) = {}, got {}'.format(
            what, ARCH_LAGS_MAX, top, n_lags))
    return int(n_obs), int(n_lags)


def sim_arch(params, n_obs=100, n_lags=5, seed=0, offset=0, want_data=False, want_summaries=True):
    """ARCH(1) simulator on the device (elfi/examples/arch.py:65-132).  params: (batch, 2) columns
    t1, t2.  Row i is a pure function of (seed, offset + i).

    Returns (Y, S), each None unless asked for: Y (batch, n_obs) the series y_1 .. y_n, S (batch,
    arch_nsumm(n_lags)) its summaries [MU, VAR, AC_1 .. AC_L, PW in itertools.combinations order],
    computed in the simulator without writing Y, bit for bit :func:`arch_summaries` of Y."""
    n_obs, n_lags = _arch_shape(n_obs, n_lags, 'the device ARCH simulator and its summaries')
    P = _params(params, 'ARCH', ('t1', 't2'))
    B = P.shape[0]
    K = arch_nsumm(n_lags)
    Y = dev.empty((B, n_obs)) if want_data else None
    S = dev.empty((B, K)) if want_summaries else None
    _lib.call('elfi_b200_sim_arch_f64', dev.context(), dev.ptr(P), _ld(P), B, n_obs, n_lags,
              int(seed), int(offset), dev.ptr(Y), n_obs, dev.ptr(S), K, dev.stream_ptr())
    return Y, S


def arch_summaries(y, n_lags=5):
    """The ARCH summaries of elfi/examples/arch.py:135-208 for each row of device data y (batch, n),
    any strides (the reference's y[:, 1:] view included): a (batch, arch_nsumm(n_lags)) tensor
    [MU, VAR, AC_1 .. AC_L, PW_i_j in itertools.combinations order], bit for bit NumPy's."""
    y = _data(y, 'arch_summaries', ('batch', 'n'))
    B = int(y.shape[0])
    n, n_lags = _arch_shape(int(y.shape[1]), n_lags, 'the device ARCH summaries')
    K = arch_nsumm(n_lags)
    S = dev.empty((B, K))
    _lib.call('elfi_b200_arch_summaries_f64', dev.context(), dev.ptr(y), y.stride(0), y.stride(1),
              B, n, n_lags, dev.ptr(S), K, dev.stream_ptr())
    return S


# ---- AR(1) model (elfi/examples/ar1.py) -----------------------------------------------------------
AR1_NOBS_MAX = _lib.CONSTANTS['AR1_NOBS_MAX']
AR1_BATCH_MAX = _lib.CONSTANTS['AR1_BATCH_MAX']


def sim_ar1(phi, n_obs=200, seed=0, offset=0, obs=None, thresholds=None, want_data=None):
    """AR(1) simulator on the device (elfi/examples/ar1.py:11-38): x_t = phi x_{t-1} + w_t, x_0 = 0,
    with the Euclidean distance to an observed series fused.  phi: (batch,) or (batch, 1).  Row i
    is a pure function of (seed, offset + i).

    obs : None or the observed series, n_obs values
    thresholds : None, or one threshold (a float, a host array or a device tensor): needs obs
    want_data : write the series; None writes it only when no obs is given

    Returns (X, d, idx): X (batch, n_obs) the series x_1 .. x_n (None unless want_data), d (batch,)
    the distance of each series to obs (None without obs), bit for bit :func:`dist_euclid` of X,
    and idx the ascending indices of the rows with d <= threshold (None without thresholds), as
    :func:`dist_euclid` returns them.  The distance is computed without writing X.
    1 <= n_obs <= AR1_NOBS_MAX, batch <= AR1_BATCH_MAX."""
    if int(n_obs) != n_obs or not 1 <= n_obs <= AR1_NOBS_MAX:
        raise ValueError('the device AR(1) simulator takes an integer 1 <= n_obs <= {}, got '
                         '{}'.format(AR1_NOBS_MAX, n_obs))
    n_obs = int(n_obs)
    P = _params(phi, 'AR(1)', ('phi',))
    B = P.shape[0]
    if B > AR1_BATCH_MAX:
        raise ValueError('the device AR(1) simulator takes at most {} rows per call, got '
                         '{}'.format(AR1_BATCH_MAX, B))
    if thresholds is not None and obs is None:
        raise ValueError('thresholds need the observed series obs')
    if want_data is None:
        want_data = obs is None
    if not want_data and obs is None:
        raise ValueError('sim_ar1 asked for neither the data nor a distance')
    phi_t = P[:, 0].contiguous()
    obs_t = thr = d = acc_idx = n_acc = None
    if obs is not None:
        obs_t = _dist_obs(obs, n_obs)
        thr = _dist_thresholds(thresholds, 1, device_thresholds=True)
        d = dev.empty((B,))
        if thr is not None:
            n_acc = dev.zeros((1,), dtype=torch.int64)
            acc_idx = dev.empty((max(B, 1),), dtype=torch.int32)
    thr_on_device = dev.is_device_array(thr)
    X = dev.empty((B, n_obs)) if want_data else None
    _lib.call('elfi_b200_sim_ar1_f64', dev.context(), dev.ptr(phi_t), B, n_obs, int(seed),
              int(offset), dev.ptr(X), n_obs, dev.ptr(obs_t),
              None if thr_on_device else dev.ptr(thr), dev.ptr(thr) if thr_on_device else None,
              dev.ptr(d), dev.ptr(acc_idx), dev.ptr(n_acc), dev.stream_ptr())
    return X, d, _dist_accepted(acc_idx, n_acc)


# ---- n-D Gaussian mean model (elfi/examples/gauss.py, nd_mean=True) -------------------------------
GAUSS_ND_D_MAX = _lib.CONSTANTS['GAUSS_ND_D_MAX']
GAUSS_ND_NOBS_MAX = _lib.CONSTANTS['GAUSS_ND_NOBS_MAX']
GAUSS_ND_SUMM_NOBS_MAX = _lib.CONSTANTS['GAUSS_ND_SUMM_NOBS_MAX']


def gauss_nd_summaries(y, out=None):
    """np.mean(y, axis=1) and np.var(y, axis=1) of (batch, n, D) data (elfi/examples/gauss.py:142-173)
    as one (batch, 2 D) tensor [means | variances], bit for bit NumPy's on the C-contiguous array:
    each coordinate's sum over the n observations is NumPy's pairwise sum for D = 1 and a left fold
    for D >= 2.  Device float64 data is read in place, whatever its strides."""
    y = _data(y, 'gauss_nd_summaries', ('batch', 'n', 'D'))
    B, n, D = (int(v) for v in y.shape)
    if not 1 <= n <= GAUSS_ND_SUMM_NOBS_MAX or D < 1:
        raise ValueError('gauss_nd_summaries takes 1 <= n <= {} observations of D >= 1 coordinates, '
                         'got shape {}'.format(GAUSS_ND_SUMM_NOBS_MAX, tuple(y.shape)))
    out = _out(out, (B, 2 * D), 'gauss_nd_summaries')
    _lib.call('elfi_b200_gauss_nd_summaries_f64', dev.context(), dev.ptr(y), y.stride(0),
              y.stride(1), y.stride(2), B, n, D, dev.ptr(out), out.stride(0) if B > 1 else 2 * D,
              dev.stream_ptr())
    return out


def gauss_nd_distance(S, obs):
    """The reference's euclidean_multidim (elfi/examples/gauss.py:176-198) on the device:
    sqrt(np.sum((S - obs)**2., axis=1)) of S (batch, D), any strides, and the observed row obs
    (D values), bit for bit NumPy's (one pairwise sum per row).  Returns d (batch,)."""
    S = _data(S, 'gauss_nd_distance', ('batch', 'D'))
    B, D = (int(v) for v in S.shape)
    if not 1 <= D <= GAUSS_ND_SUMM_NOBS_MAX:
        raise ValueError('gauss_nd_distance takes 1 <= D <= {} columns, got shape {}'.format(
            GAUSS_ND_SUMM_NOBS_MAX, tuple(S.shape)))
    obs_t = _dist_obs(obs, D)
    d = dev.empty((B,))
    _lib.call('elfi_b200_gauss_nd_distance_f64', dev.context(), dev.ptr(S), S.stride(0),
              S.stride(1), B, D, dev.ptr(obs_t), dev.ptr(d), dev.stream_ptr())
    return d


def gauss_nd_factor(cov_matrix, D):
    """The (D, D) factor A = sqrt(s)[:, None] * vh of NumPy's RandomState.multivariate_normal for
    the covariance SciPy's multivariate_normal makes of cov_matrix (None: the identity; a scalar:
    that multiple of it; a vector: its diagonal), so that mean + z @ A has the reference's law.  A
    covariance that is not symmetric positive semidefinite raises, as SciPy does."""
    cov = np.asarray(1.0 if cov_matrix is None else cov_matrix, dtype=np.float64)
    if cov.ndim == 0:
        cov = cov * np.eye(D)
    elif cov.ndim == 1:
        cov = np.diag(cov)
    if cov.shape != (D, D):
        raise ValueError('the covariance of {} means must be ({}, {}), got shape {}'.format(
            D, D, D, cov.shape))
    if not np.all(np.isfinite(cov)):
        raise ValueError('the covariance must be finite')
    _, s, vh = np.linalg.svd(cov)
    tol = 1e-8
    if not np.allclose(np.dot(vh.T * s, vh), cov, rtol=tol, atol=tol):
        raise ValueError('the covariance must be symmetric positive semidefinite')
    return np.ascontiguousarray(np.sqrt(s)[:, None] * vh)


def _gauss_nd_means(mu):
    """(batch, D) device means: a matrix, or D device or host columns of one length."""
    if dev.is_device_array(mu) and mu.dtype == torch.float64 and mu.dim() == 2:
        return mu
    if isinstance(mu, (list, tuple)):
        cols = [dev.to_device(c).reshape(-1) for c in mu]
        if len({int(c.shape[0]) for c in cols}) != 1:
            raise ValueError('the mean columns must have one length, got {}'.format(
                [int(c.shape[0]) for c in cols]))
        return torch.stack(cols, 1)
    return _data(mu, 'sim_gauss_nd', ('batch', 'D'))


def sim_gauss_nd(mu, A, n_obs=15, seed=0, offset=0, want_data=False, want_summaries=True):
    """The n-D Gaussian mean simulator on the device (elfi/examples/gauss.py:38-72): row i draws
    n_obs observations y_t = mu_i + z_t @ A, z_t standard normal (Philox streams; statistical parity
    with the reference's SciPy draws).  Row i is a pure function of (seed, offset + i).

    mu : (batch, D) device matrix (any strides) or D columns, 1 <= D <= GAUSS_ND_D_MAX
    A : (D, D) factor, gauss_nd_factor(cov_matrix, D)
    Returns (Y, S), each None unless asked for: Y (batch, n_obs, D) the data, S (batch, 2 D) its
    summaries [means | variances], computed without writing Y, bit for bit
    :func:`gauss_nd_summaries` of Y.  1 <= n_obs <= GAUSS_ND_NOBS_MAX."""
    M = _gauss_nd_means(mu)
    B, D = (int(v) for v in M.shape)
    if not 1 <= D <= GAUSS_ND_D_MAX:
        raise ValueError('the device n-D Gaussian simulator takes 1 <= D <= {} means, got shape '
                         '{}'.format(GAUSS_ND_D_MAX, tuple(M.shape)))
    if int(n_obs) != n_obs or not 1 <= n_obs <= GAUSS_ND_NOBS_MAX:
        raise ValueError('the device n-D Gaussian simulator takes an integer 1 <= n_obs <= {}, got '
                         '{}'.format(GAUSS_ND_NOBS_MAX, n_obs))
    n_obs = int(n_obs)
    A = np.ascontiguousarray(dev.to_host(A) if dev.is_device_array(A) else A, dtype=np.float64)
    if A.shape != (D, D):
        raise ValueError('the factor of {} means must be ({}, {}), got shape {}'.format(
            D, D, D, A.shape))
    if not (want_data or want_summaries):
        raise ValueError('sim_gauss_nd asked for neither the data nor the summaries')
    Y = dev.empty((B, n_obs, D)) if want_data else None
    S = dev.empty((B, 2 * D)) if want_summaries else None
    _lib.call('elfi_b200_sim_gauss_nd_f64', dev.context(), dev.ptr(M), M.stride(0), M.stride(1),
              B, D, dev.ptr(A), n_obs, int(seed), int(offset), dev.ptr(Y), n_obs * D, dev.ptr(S),
              2 * D, dev.stream_ptr())
    return Y, S


# ---- M/G/1 queue (elfi/examples/mg1.py) ------------------------------------------------------------
MG1_NOBS_MIN = _lib.CONSTANTS['MG1_NOBS_MIN']
MG1_NOBS_MAX = _lib.CONSTANTS['MG1_NOBS_MAX']
MG1_NQ_MAX = _lib.CONSTANTS['MG1_NQ_MAX']


def _mg1_q(q):
    q = np.array(q, dtype=np.float64).reshape(-1)
    if not 1 <= q.size <= MG1_NQ_MAX:
        raise ValueError('the device quantiles take 1 <= len(q) <= {} levels, got {}'.format(
            MG1_NQ_MAX, q.size))
    if not np.all((q >= 0) & (q <= 1)):
        raise ValueError('the quantile levels q must lie in [0, 1]')
    return np.ascontiguousarray(q)


def _mg1_n(n, what):
    if int(n) != n or not MG1_NOBS_MIN <= n <= MG1_NOBS_MAX:
        raise ValueError('{} take {} <= n <= {} observations per row, got {}'.format(
            what, MG1_NOBS_MIN, MG1_NOBS_MAX, n))
    return int(n)


def sim_mg1(params, n_obs=50, q=np.linspace(0, 1, 10), seed=0, offset=0, want_data=False,
            want_summaries=True):
    """M/G/1 queue simulator on the device (elfi/examples/mg1.py:21-54).  params: (batch, 3) columns
    t1, t2, t3.  Row i is a pure function of (seed, offset + i); rows where the reference raises
    (1/t3 with its sign bit set, t2 - t1 not finite) are NaN.

    Returns (Y, S), each None unless asked for: Y (batch, n_obs) the inter-departure times, S
    (batch, len(q)) their quantiles np.quantile(y, q) (method 'linear'), computed in the simulator
    without writing Y, bit for bit :func:`row_quantiles` of Y."""
    n_obs = _mg1_n(n_obs, 'the device M/G/1 simulator and its quantiles')
    qv = _mg1_q(q)
    P = _params(params, 'M/G/1', ('t1', 't2', 't3'))
    B = P.shape[0]
    Y = dev.empty((B, n_obs)) if want_data else None
    S = dev.empty((B, qv.size)) if want_summaries else None
    _lib.call('elfi_b200_sim_mg1_f64', dev.context(), dev.ptr(P), _ld(P), B, n_obs, qv.size,
              dev.ptr(qv), int(seed), int(offset), dev.ptr(Y), n_obs, dev.ptr(S), qv.size,
              dev.stream_ptr())
    return Y, S


def row_quantiles(x, q):
    """np.quantile(x, q, axis=1).T (method 'linear') of device data x (batch, n), any strides:
    a (batch, len(q)) tensor, bit for bit NumPy's; a row containing NaN has every quantile NaN.
    Limits: 2 <= n <= MG1_NOBS_MAX, 1 <= len(q) <= MG1_NQ_MAX, q in [0, 1]."""
    x = _data(x, 'row_quantiles', ('batch', 'n'))
    n = _mg1_n(int(x.shape[1]), 'the device row quantiles')
    qv = _mg1_q(q)
    B = int(x.shape[0])
    S = dev.empty((B, qv.size))
    _lib.call('elfi_b200_row_quantiles_f64', dev.context(), dev.ptr(x), x.stride(0), x.stride(1),
              B, n, qv.size, dev.ptr(qv), dev.ptr(S), qv.size, dev.stream_ptr())
    return S


# ---- alpha-stable stochastic volatility model (elfi/examples/stochastic_volatility_model.py) ---------
SVM_NPARAMS = 7               # alpha, beta, kappa, eta, mu, phi, sigma
SVM_LEVELS = (0.05, 0.25, 0.5, 0.75, 0.95)


def sim_svm(params, n_obs=50, seed=0, offset=0, want_data=False, want_summaries=True):
    """Alpha-stable stochastic volatility simulator on the device
    (elfi/examples/stochastic_volatility_model.py).  params: (batch, 7) columns alpha, beta, kappa,
    eta, mu, phi, sigma.  Row i is a pure function of (seed, offset + i); rows where the reference
    raises (levy_stable's argcheck, kappa < 0, sigma < 0, phi NaN) are NaN.

    Returns (Y, S), each None unless asked for: Y (batch, n_obs) the observations, S (batch, 2)
    their quantile kurtosis and skewness [kurt, skew], computed in the simulator without writing
    Y, bit for bit :func:`svm_summaries` of Y."""
    n_obs = _mg1_n(n_obs, 'the device stochastic volatility simulator and its summaries')
    P = _params(params, 'stochastic volatility',
                ('alpha', 'beta', 'kappa', 'eta', 'mu', 'phi', 'sigma'))
    B = P.shape[0]
    Y = dev.empty((B, n_obs)) if want_data else None
    S = dev.empty((B, 2)) if want_summaries else None
    _lib.call('elfi_b200_sim_svm_f64', dev.context(), dev.ptr(P), _ld(P), B, n_obs, int(seed),
              int(offset), dev.ptr(Y), n_obs, dev.ptr(S), 2, dev.stream_ptr())
    return Y, S


def svm_summaries(x):
    """[kurt, skew] (batch, 2) of device data x (batch, n), any strides, without the fused kernel:
    :func:`row_quantiles` at 0.05, 0.25, 0.5, 0.75, 0.95, then the reference's subtractions and
    division in fp64 (IEEE, so NumPy's bits):
    kurt = (q95 - q05) / (q75 - q25), skew = ((q95 - q50) - (q50 - q05)) / (q95 - q05)."""
    q = row_quantiles(x, SVM_LEVELS)
    q05, q25, q50, q75, q95 = q.unbind(1)
    kurt = (q95 - q05) / (q75 - q25)
    skew = ((q95 - q50) - (q50 - q05)) / (q95 - q05)
    return torch.stack([kurt, skew], dim=1)


# ---- scratch assay (elfi/examples/scratch_assay.py) -----------------------------------------------
SA_SITES_MAX = _lib.CONSTANTS['SA_SITES_MAX']
SA_ITER_MAX = _lib.CONSTANTS['SA_ITER_MAX']
SA_BATCH_MAX = _lib.CONSTANTS['SA_BATCH_MAX']


def scratch_assay_steps(obs_period=12, obs_interval=1 / 12, tau=1 / 24):
    """(num_iter, interval, num_obs) as the reference's cell_sim computes them:
    int(obs_period / tau), int(obs_interval / tau) and int(num_iter / interval)."""
    num_iter = int(obs_period / tau)
    interval = int(obs_interval / tau)
    if not 0 <= num_iter <= SA_ITER_MAX:
        raise ValueError('the device scratch assay simulator takes 0 <= int(obs_period / tau) < '
                         '2^31 iterations, got {}'.format(num_iter))
    if interval < 1:
        raise ValueError('the scratch assay simulator takes obs_interval >= tau (at least one '
                         'iteration between observations), got int(obs_interval / tau) = '
                         '{}'.format(interval))
    return num_iter, interval, int(num_iter / interval)


def _scratch_init(init_arr):
    """The initial lattice as a contiguous (nrows, ncols) uint8 device tensor, checked."""
    t = init_arr if dev.is_device_array(init_arr) else dev.to_device(
        np.asarray(init_arr, dtype=np.float64))
    if t.dim() != 2:
        raise ValueError('init_arr must be a 2-d (nrows, ncols) lattice, got shape {}'.format(
            tuple(t.shape)))
    nrows, ncols = (int(v) for v in t.shape)
    if not (1 <= nrows and 1 <= ncols and nrows * ncols <= SA_SITES_MAX):
        raise ValueError('the device scratch assay simulator takes a lattice of 1 to {} sites, '
                         'got {} x {}'.format(SA_SITES_MAX, nrows, ncols))
    if not bool(torch.all((t == 0) | (t == 1))):
        raise ValueError('init_arr must hold 0s and 1s only')
    return (t != 0).to(torch.uint8).contiguous()


def sim_scratch_assay(params, init_arr, obs_period=12, obs_interval=1 / 12, tau=1 / 24, seed=0,
                      offset=0, want_data=False, want_summaries=True):
    """Scratch assay simulator on the device (elfi/examples/scratch_assay.py, Johnston et al.
    2014), its streams replayed exactly by tests/scratch_assay_replay.py.  params: (batch, 2)
    columns pm, pp; init_arr: the (nrows, ncols) initial lattice of 0s and 1s, at most
    SA_SITES_MAX sites.  The iteration and observation counts are the reference's
    (:func:`scratch_assay_steps`).  Row i is a pure function of (seed, offset + i).

    Returns (X, S), each None unless asked for: X (batch, nrows, ncols, num_obs + 1) bool, the
    frames; S (batch, num_obs + 1) float64, the mismatches between consecutive frames and the
    final cell count (the reference's cell_summaries), computed in the simulator without writing
    X, equal to :func:`scratch_assay_summaries` of X."""
    num_iter, interval, num_obs = scratch_assay_steps(obs_period, obs_interval, tau)
    init = _scratch_init(init_arr)
    nrows, ncols = (int(v) for v in init.shape)
    P = _params(params, 'scratch assay', ('pm', 'pp'))
    B = P.shape[0]
    if B > SA_BATCH_MAX:
        raise ValueError('the device scratch assay simulator takes at most {} rows per call, got '
                         '{}'.format(SA_BATCH_MAX, B))
    X = dev.empty((B, nrows, ncols, num_obs + 1), dtype=torch.bool) if want_data else None
    S = dev.empty((B, num_obs + 1)) if want_summaries else None
    _lib.call('elfi_b200_sim_scratch_assay_f64', dev.context(), dev.ptr(P), _ld(P), B,
              dev.ptr(init), nrows, ncols, num_iter, interval, int(seed), int(offset), dev.ptr(S),
              num_obs + 1, dev.ptr(X), dev.stream_ptr())
    return X, S


def scratch_assay_summaries(x):
    """The reference's cell_summaries of data (batch, nrows, ncols, n_frames), any strides, nonzero
    meaning a cell: a (batch, n_frames) float64 tensor of the n_frames - 1 mismatches between
    consecutive frames, then the cells of the last frame.  On 0 / 1 data these are NumPy's values
    exactly (they are integers)."""
    x = _mask(x, 'scratch_assay_summaries', ('batch', 'nrows', 'ncols', 'n_frames'))
    B, nrows, ncols, frames = (int(v) for v in x.shape)
    if min(nrows, ncols, frames) < 1:
        raise ValueError('scratch_assay_summaries takes nrows, ncols, n_frames >= 1, got shape '
                         '{}'.format(tuple(x.shape)))
    S = dev.empty((B, frames))
    _lib.call('elfi_b200_scratch_assay_summaries_f64', dev.context(), dev.ptr(x), x.stride(0),
              x.stride(1), x.stride(2), x.stride(3), B, nrows, ncols, frames, dev.ptr(S), frames,
              dev.stream_ptr())
    return S


# ---- Bayesian synthetic likelihood (elfi/methods/bsl/pdf_methods.py) ------------------------------
SYNLIK_D_MAX = _lib.CONSTANTS['SYNLIK_D_MAX']
SYNLIK_ESTIMATORS = {'standard': 0, 'unbiased': 1}


def synlik(S, y, estimator='standard', penalties=None, whitening=None):
    """Gaussian synthetic log-likelihood of the observed summaries y (d,) under each group of
    simulated summaries S, (n, d) or (G, n, d), host or device, any row and group strides.  A y of
    shape (G, d), G > 1, gives each group its own observation (any row stride, 0 included); group
    g's value is then the one S[g] alone would give against y[g].

    estimator 'standard' is gaussian_syn_likelihood (Warton shrinkage at each of the penalties, and
    whitening by the (d, d) matrix W, both optional); 'unbiased' is
    gaussian_syn_likelihood_ghurye_olkin.  Returns a device tensor (G,), or (G, K) for K penalties.
    A group whose inputs are not all finite, or whose covariance fails its Cholesky test, gives
    -inf (include/elfi_b200.h states the test).  Limits: 1 <= d <= SYNLIK_D_MAX, n >= 2."""
    if estimator not in SYNLIK_ESTIMATORS:
        raise ValueError("estimator must be 'standard' or 'unbiased', got {!r}".format(estimator))
    if estimator == 'unbiased' and (penalties is not None or whitening is not None):
        raise ValueError('the unbiased estimator takes no penalties and no whitening')
    X = S if dev.is_device_array(S) and S.dtype == torch.float64 else dev.to_device(S)
    if X.dim() == 2:
        X = X[None]
    if X.dim() != 3:
        raise ValueError('synlik takes S of shape (n, d) or (G, n, d), got {}'.format(
            tuple(X.shape)))
    G, n, d = (int(v) for v in X.shape)
    if not 1 <= d <= SYNLIK_D_MAX:
        raise ValueError('synlik takes 1 <= d <= {} summaries, got d = {}'.format(SYNLIK_D_MAX, d))
    if n < 2:
        raise ValueError('synlik takes n >= 2 simulations per group, got n = {}'.format(n))
    if X.stride(2) != 1 or X.stride(1) < d or X.stride(0) < 0:
        X = X.contiguous()
    yv = y if dev.is_device_array(y) and y.dtype == torch.float64 else dev.to_device(y)
    # d values in any shape are the one observation of every group, as before per-group rows
    per_group = yv.dim() == 2 and yv.numel() != d
    if per_group:
        if tuple(yv.shape) != (G, d):
            raise ValueError('y has shape {}, S has G = {} groups of d = {} summaries'.format(
                tuple(yv.shape), G, d))
        if yv.stride(1) != 1 or 0 < yv.stride(0) < d or yv.stride(0) < 0:
            yv = yv.contiguous()        # stride 0 (an expanded row) is kept: ld_y = 0
    else:
        yv = yv.reshape(-1).contiguous()
        if yv.numel() != d:
            raise ValueError('y has {} values, S has d = {} summaries'.format(yv.numel(), d))
    W = None
    if whitening is not None:
        W = dev.to_device(whitening).contiguous()
        if tuple(W.shape) != (d, d):
            raise ValueError('whitening must be a ({0}, {0}) matrix, got shape {1}'.format(
                d, tuple(W.shape)))
    pen, K = None, 0
    if penalties is not None:
        pen = np.ascontiguousarray(np.asarray(penalties, dtype=np.float64).reshape(-1))
        K = pen.size
        if K == 0:
            raise ValueError('penalties is empty')
        if not np.all((pen >= 0) & (pen <= 1)):
            raise ValueError('Warton penalties must lie in [0, 1], got {}'.format(pen))
    out = dev.empty((G, K) if K else (G,))
    tail = (dev.ptr(W), SYNLIK_ESTIMATORS[estimator],
            None if pen is None else ctypes.c_void_p(pen.ctypes.data), K, dev.ptr(out),
            dev.stream_ptr())
    if per_group:
        _lib.call('elfi_b200_synlik_obs_f64', dev.context(), dev.ptr(X), X.stride(1),
                  X.stride(0), G, n, d, dev.ptr(yv), yv.stride(0), *tail)
    else:
        _lib.call('elfi_b200_synlik_f64', dev.context(), dev.ptr(X), X.stride(1), X.stride(0), G,
                  n, d, dev.ptr(yv), *tail)
    return out


BSL_MAX_CHAINS = _lib.CONSTANTS['BSL_MAX_CHAINS']


def bsl_mh_tables(specs, sigma_proposals, sources=None, bounds=None):
    """The host constants of :func:`bsl_mh_step`, checked once per run: the (p, 7) prior table
    (``specs`` (p, 5) and ``sources`` (p, 2) as in :func:`prior_logpdf`), the lower Cholesky
    factor of the (p, p) proposal covariance, and the (p, 2) logit bounds or None."""
    specs = np.atleast_2d(np.asarray(specs, dtype=np.float64))
    p = specs.shape[0]
    table = _prior_table(specs, -np.ones((p, 2)) if sources is None else sources)
    cov = np.atleast_2d(np.asarray(sigma_proposals, dtype=np.float64))
    if cov.shape != (p, p):
        raise ValueError('sigma_proposals must be a ({0}, {0}) covariance, got shape {1}'.format(
            p, cov.shape))
    try:
        L = np.ascontiguousarray(np.linalg.cholesky(cov))
    except np.linalg.LinAlgError:
        raise ValueError('sigma_proposals is not positive definite') from None
    bnd = None
    if bounds is not None:
        bnd = np.ascontiguousarray(np.asarray(bounds, dtype=np.float64))
        if bnd.shape != (p, 2) or np.isnan(bnd).any():
            raise ValueError('logit_transform_bound must be ({}, 2) lower and upper bounds, got '
                             '{}'.format(p, bounds))
    return table, L, bnd


def bsl_mh_step(tables, t, loglik, prop, prop_lp, chains, logpost, n_acc, rows, seed, burn_in=0,
                lanes=None):
    """Iteration t of C lock-step BSL chains on the device (include/elfi_b200.h states the step
    and its Philox stream): the decision of every chain from the round's log-likelihoods
    ``loglik`` (C,) and the pending proposals ``prop`` (C, p) with their log priors ``prop_lp``
    (C,), written to row t of ``chains`` (C, n_samples, p) and ``logpost`` (C, n_samples) and
    counted in ``n_acc`` (C,) int64 from ``burn_in``; then, unless t is the last iteration, the
    proposals of iteration t + 1 into ``prop`` / ``prop_lp`` and the next batch's parameters into
    ``rows`` (p, C b), chain c's block in columns [c b, (c + 1) b).  ``tables`` is
    :func:`bsl_mh_tables`.  ``seed`` is an int (every chain's Philox key, chain c on lane c), or
    a (C,) int64 device tensor of per-chain keys with ``lanes`` an optional (C,) integer device
    tensor of lanes (default 0 .. C - 1), so that the chains of several samplers step in one
    launch.  Asynchronous; nothing is read back."""
    table, L, bnd = tables
    C, n_samples, p = (int(v) for v in chains.shape)
    if not 1 <= C <= BSL_MAX_CHAINS:
        raise ValueError('1 <= C <= 2^22 chains, got {}'.format(C))
    if p != L.shape[0] or rows.dim() != 2 or rows.shape[0] != p or rows.shape[1] % C \
            or rows.stride(1) != 1:
        raise ValueError('rows must be a ({}, C b) array with contiguous columns'.format(p))
    for name, x, shape, dtype in (('loglik', loglik, (C,), torch.float64),
                                  ('prop', prop, (C, p), torch.float64),
                                  ('prop_lp', prop_lp, (C,), torch.float64),
                                  ('chains', chains, (C, n_samples, p), torch.float64),
                                  ('logpost', logpost, (C, n_samples), torch.float64),
                                  ('n_acc', n_acc, (C,), torch.int64)):
        if not dev.is_device_array(x) or tuple(x.shape) != shape or x.dtype != dtype \
                or not x.is_contiguous():
            raise ValueError('{} must be a contiguous {} device array of shape {}'.format(
                name, dtype, shape))
    tail = (dev.ptr(table), dev.ptr(L), dev.ptr(bnd), dev.ptr(loglik), dev.ptr(prop),
            dev.ptr(prop_lp), dev.ptr(chains), dev.ptr(logpost), dev.ptr(n_acc), dev.ptr(rows),
            rows.stride(0), dev.stream_ptr())
    b = int(rows.shape[1]) // C
    if not dev.is_device_array(seed):
        if lanes is not None:
            raise ValueError('lanes go with per-chain keys: a (C,) int64 device tensor seed')
        _lib.call('elfi_b200_bsl_mh_step_f64', dev.context(), C, p, int(t), n_samples,
                  int(burn_in), b, int(seed), *tail)
        return
    if tuple(seed.shape) != (C,) or seed.dtype != torch.int64:
        raise ValueError('keys (seed) must be a ({},) int64 device tensor, got {} {}'.format(
            C, tuple(seed.shape), seed.dtype))
    keys = seed.contiguous()
    if lanes is None:
        lanes = torch.arange(C, dtype=torch.int32, device=keys.device)
    elif not dev.is_device_array(lanes) or tuple(lanes.shape) != (C,) or \
            lanes.dtype not in (torch.int32, torch.int64):
        raise ValueError('lanes must be a ({},) int32 or int64 device tensor'.format(C))
    lanes = lanes.to(torch.int32).contiguous()      # the bits of uint32 lanes
    _lib.call('elfi_b200_bsl_mh_step_keyed_f64', dev.context(), C, p, int(t), n_samples,
              int(burn_in), b, dev.ptr(keys), dev.ptr(lanes), *tail)


# ---- BOLFIRE ratio-estimation classifier (elfi/methods/classifier.py) ------------------------------
LOGREG_D_MAX = _lib.CONSTANTS['LOGREG_D_MAX']
LOGREG_PENALTIES = {'l1': 0, 'l2': 1}
LOGREG_HEAD = _lib.CONSTANTS['LOGREG_HEAD']
LOGREG_STATUS = {1: 'converged', 0: 'not converged', -1: 'bad labels', -2: 'non-finite input'}


def logreg_block_size(d):
    """Doubles of the device fit block of a d-feature logistic regression."""
    return LOGREG_HEAD + 3 * int(d)


class LogRegFit:
    """A logistic-regression fit on the device: `block` is the (LOGREG_HEAD + 3 d,) result block of
    elfi_b200_logreg_fit_f64 (intercept, n_iter, status, objective, subgradient norm, then mean_,
    scale_ and coef_).  `host()` reads it once and keeps the host copy."""

    def __init__(self, block, d, penalty, C):
        self.block, self.d, self.penalty, self.C = block, int(d), penalty, float(C)
        self._host = None

    def set_host(self, values):
        """Record the block's host values, read together with something else."""
        self._host = np.asarray(values, dtype=np.float64)[:logreg_block_size(self.d)]

    def host(self):
        if self._host is None:
            self._host = dev.to_host(self.block).astype(np.float64)
        return self._host

    def _part(self, k):
        h = self.host()
        return h[LOGREG_HEAD + k * self.d:LOGREG_HEAD + (k + 1) * self.d]

    @property
    def intercept_(self):
        return float(self.host()[0])

    @property
    def n_iter(self):
        return int(self.host()[1])

    @property
    def status(self):
        return int(self.host()[2])

    @property
    def converged(self):
        return self.status == 1

    @property
    def objective(self):
        return float(self.host()[3])

    @property
    def subgradient_norm(self):
        return float(self.host()[4])

    @property
    def mean_(self):
        return self._part(0)

    @property
    def scale_(self):
        return self._part(1)

    @property
    def coef_(self):
        return self._part(2)

    def check(self):
        """ValueError for a fit the device rejected (labels, or non-finite values in X)."""
        s = self.status
        if s == -1:
            raise ValueError('logreg_fit: the labels must be +1 or -1 with both classes present')
        if s == -2:
            raise ValueError('logreg_fit: X contains NaN or infinity, or a value too large for '
                             'float64')
        return self


def _logreg_rows(X, name):
    X = _matrix(X)
    if X.shape[0] > 1 and X.stride(0) < X.shape[1]:
        X = X.contiguous()
    return X


def logreg_fit(X, y, penalty='l1', C=1.0, max_iter=100, out=None):
    """Fit the reference's ratio-estimation classifier (StandardScaler, then liblinear's L1- or
    L2-penalised logistic regression with a penalised intercept) to the optimum on the device.
    X is (n, d) with any row stride, y holds n labels +1 / -1; host or device.  Returns a LogRegFit
    whose block stays on the device (`out`, of logreg_block_size(d) doubles, if given).  Host
    labels are checked here; device labels are checked by the kernel and reported when the block
    is read (LogRegFit.check)."""
    if penalty not in LOGREG_PENALTIES:
        raise ValueError("penalty must be 'l1' or 'l2', got {!r}".format(penalty))
    C = float(C)
    if not (C > 0 and np.isfinite(C)):
        raise ValueError('C must be positive and finite, got {}'.format(C))
    if int(max_iter) != max_iter or max_iter < 0:
        raise ValueError('max_iter must be a non-negative integer, got {}'.format(max_iter))
    if not dev.is_device_array(y):
        yh = np.asarray(y, dtype=np.float64).reshape(-1)
        if not np.all((yh == 1) | (yh == -1)):
            raise ValueError('logreg_fit takes labels +1 and -1')
        if np.all(yh == 1) or np.all(yh == -1):
            raise ValueError('logreg_fit needs samples of both classes, got only {}'.format(
                yh[0] if yh.size else 'none'))
    Xd = _logreg_rows(X, 'X')
    n, d = int(Xd.shape[0]), int(Xd.shape[1])
    if not 1 <= d <= LOGREG_D_MAX:
        raise ValueError('logreg_fit takes 1 <= d <= {} features, got d = {}'.format(
            LOGREG_D_MAX, d))
    if n < 2:
        raise ValueError('logreg_fit takes n >= 2 rows, got n = {}'.format(n))
    yd = y if dev.is_device_array(y) else dev.to_device(yh)
    yd = yd.reshape(-1)
    if yd.dtype != torch.float64 or not yd.is_contiguous():
        yd = yd.to(torch.float64).contiguous()
    if yd.numel() != n:
        raise ValueError('y has {} labels, X has {} rows'.format(yd.numel(), n))
    block = dev.empty((logreg_block_size(d),)) if out is None else out
    if block.numel() != logreg_block_size(d) or not block.is_contiguous():
        raise ValueError('out must be a contiguous device buffer of {} doubles'.format(
            logreg_block_size(d)))
    _lib.call('elfi_b200_logreg_fit_f64', dev.context(), dev.ptr(Xd), _ld(Xd), n, d, dev.ptr(yd),
              LOGREG_PENALTIES[penalty], C, int(max_iter), dev.ptr(block), dev.stream_ptr())
    return LogRegFit(block, d, penalty, C)


def logreg_predict(fit, X, class_min=0.0, out=None):
    """log(p / (1 - p)) per row of X (m, d), p = max(expit(decision value), class_min): the
    reference's predict_log_likelihood_ratio, as a device tensor (m,) (`out` if given).  A row
    with a non-finite value, or a fit the device rejected, gives NaN."""
    if not isinstance(fit, LogRegFit):
        raise ValueError('logreg_predict takes the LogRegFit of logreg_fit')
    Xd = _logreg_rows(X, 'X')
    m, d = int(Xd.shape[0]), int(Xd.shape[1])
    if d != fit.d:
        raise ValueError('X has {} features per row, the fit {}'.format(d, fit.d))
    res = dev.empty((m,)) if out is None else out
    if res.numel() != m or not res.is_contiguous():
        raise ValueError('out must be a contiguous device buffer of {} doubles'.format(m))
    _lib.call('elfi_b200_logreg_predict_f64', dev.context(), dev.ptr(fit.block), d, dev.ptr(Xd),
              _ld(Xd), m, float(class_min), dev.ptr(res), dev.stream_ptr())
    return res


# ---- summary-statistic selection (TwoStageSelection, elfi/methods/diagnostics.py) ---------------
SUBSET_METRIC_CODES = {k: v for k, v in _METRICS.items() if v <= _METRICS['chebyshev']}
SUBSET_MAX_WIDTH = _lib.CONSTANTS['SUBSET_MAX_WIDTH']
SUBSET_MAX_COMBINATIONS = _lib.CONSTANTS['SUBSET_MAX_COMBINATIONS']
KNN_MAX_Q = _lib.CONSTANTS['KNN_MAX_Q']
KNN_MAX_K = _lib.CONSTANTS['KNN_MAX_K']
KNN_MAX_N = _lib.CONSTANTS['KNN_MAX_N']
KNN_MAX_SETS = _lib.CONSTANTS['KNN_MAX_SETS']


class SubsetLayout:
    """The candidate combinations of :func:`subset_distance`, checked and uploaded once: each
    combination is an ordered list of column ranges (col, width) of a (B, width) summary matrix."""

    def __init__(self, combinations, width):
        width = int(width)
        if not 1 <= width <= SUBSET_MAX_WIDTH:
            raise ValueError('subset_distance takes 1 <= {} summary columns, got {}'.format(
                SUBSET_MAX_WIDTH, width))
        combinations = [list(c) for c in combinations]
        if not 1 <= len(combinations) <= SUBSET_MAX_COMBINATIONS:
            raise ValueError('subset_distance takes 1 to {} combinations, got {}'.format(
                SUBSET_MAX_COMBINATIONS, len(combinations)))
        ranges, offsets = [], [0]
        for comb in combinations:
            if not comb:
                raise ValueError('a combination needs at least one column range')
            for col, w in comb:
                if not (w >= 1 and col >= 0 and col + w <= width):
                    raise ValueError('column range ({}, {}) outside the {} summary columns'.format(
                        col, w, width))
                ranges.append((int(col), int(w)))
            offsets.append(len(ranges))
        self.width = width
        self.n_combinations = len(combinations)
        self.ranges = dev.to_device(np.asarray(ranges, dtype=np.int32).reshape(-1, 2),
                                    dtype=torch.int32)
        self.offsets = dev.to_device(np.asarray(offsets, dtype=np.int32), dtype=torch.int32)


def subset_distance(S, obs, layout, metric='euclidean', out=None):
    """cdist of every combination of ``layout`` (a :class:`SubsetLayout`) at once: row c of the
    (C, B) result is cdist(X_c, obs_c, metric), X_c and obs_c the concatenated column ranges of
    combination c, bit for bit ('euclidean', 'sqeuclidean', 'cityblock' or 'chebyshev').  `out` may
    be a (C, >= B) device matrix with unit column stride."""
    if metric not in SUBSET_METRIC_CODES:
        raise ValueError('subset_distance takes the metrics {}, got {!r}'.format(
            ', '.join(SUBSET_METRIC_CODES), metric))
    S = _matrix(S)
    B, W = int(S.shape[0]), int(S.shape[1])
    if W != layout.width:
        raise ValueError('S has {} columns, the layout {}'.format(W, layout.width))
    obs_t = dev.to_device(obs).reshape(-1)
    if obs_t.numel() != W:
        raise ValueError('obs has {} values, S has {} columns'.format(obs_t.numel(), W))
    C = layout.n_combinations
    if out is None:
        out = dev.empty((C, B))
    if tuple(out.shape[:1]) != (C,) or out.dim() != 2 or out.shape[1] < B or \
            (B and out.stride(1) != 1):
        raise ValueError('out must be a ({}, >= {}) device matrix'.format(C, B))
    _lib.call('elfi_b200_subset_distance_f64', dev.context(), SUBSET_METRIC_CODES[metric],
              dev.ptr(S), _ld(S), B, W, dev.ptr(obs_t), dev.ptr(layout.ranges),
              dev.ptr(layout.offsets), C, dev.ptr(out), max(out.stride(0), B), dev.stream_ptr())
    return out


def _point_sets(X, name):
    """X (C, n, q) or (n, q) as a contiguous (C, n, q) float64 device array."""
    if not (dev.is_device_array(X) and X.dtype == torch.float64):
        X = dev.to_device(X)
    if X.dim() == 2:
        X = X[None]
    if X.dim() != 3:
        raise ValueError('{} takes (sets, points, dim) or (points, dim) data, got shape {}'.format(
            name, tuple(X.shape)))
    return X.contiguous()


def knn_entropy(X, k):
    """The k-th nearest-neighbour radii of C point sets and their log sums (the device part of
    diagnostics.py:214-253).  X (C, n, q) or (n, q).  Returns (R (C, n), logsum (C,)): R[c, i] is
    cKDTree(X[c]).query(X[c, i], k)[0][-1] and logsum[c] = sum_i log R[c, i] in a fixed order."""
    X = _point_sets(X, 'knn_entropy')
    C, n, q = (int(s) for s in X.shape)
    k = int(k)
    if not 1 <= q <= KNN_MAX_Q:
        raise ValueError('knn_entropy takes 1 <= q <= {} dimensions, got {}'.format(KNN_MAX_Q, q))
    if not 1 <= k <= KNN_MAX_K:
        raise ValueError('knn_entropy takes 1 <= k <= {}, got {}'.format(KNN_MAX_K, k))
    if not 1 <= n <= KNN_MAX_N:
        raise ValueError('knn_entropy takes 1 <= n <= {} points per set, got {}'.format(
            KNN_MAX_N, n))
    if not 1 <= C <= KNN_MAX_SETS:
        raise ValueError('knn_entropy takes 1 to {} sets, got {}'.format(KNN_MAX_SETS, C))
    R = dev.empty((C, n))
    logsum = dev.empty((C,))
    _lib.call('elfi_b200_knn_entropy_f64', dev.context(), dev.ptr(X), q, C, n, q, k, dev.ptr(R),
              dev.ptr(logsum), dev.stream_ptr())
    return R, logsum


def mrsse(T, P, out=None):
    """Mean root sum of squared errors of C parameter sets against m 'closest' parameter vectors
    (diagnostics.py:255-289): out[c] = mean_j ||T[c] - P[j]||_F.  T (C, n, q) or (n, q), P (m, q).
    Returns a (C,) device array (`out` if given)."""
    T = _point_sets(T, 'mrsse')
    C, n, q = (int(s) for s in T.shape)
    Pd = _matrix(P)
    m = int(Pd.shape[0])
    if not 1 <= q <= KNN_MAX_Q:
        raise ValueError('mrsse takes 1 <= q <= {} dimensions, got {}'.format(KNN_MAX_Q, q))
    if int(Pd.shape[1]) != q:
        raise ValueError('P has {} columns, the sets {}'.format(int(Pd.shape[1]), q))
    if n < 1 or m < 1 or C < 1:
        raise ValueError('mrsse needs at least one set, one point and one closest vector')
    res = dev.empty((C,)) if out is None else out
    if res.numel() != C or not res.is_contiguous():
        raise ValueError('out must be a contiguous device buffer of {} doubles'.format(C))
    _lib.call('elfi_b200_mrsse_f64', dev.context(), dev.ptr(T), q, C, n, q, dev.ptr(Pd), _ld(Pd),
              m, dev.ptr(res), dev.stream_ptr())
    return res


# ---- robust optimisation Monte Carlo (ROMC, elfi/methods/inference/romc.py) ---------------------
ROMC_MAX_P = _lib.CONSTANTS['ROMC_MAX_P']
ROMC_NM_INTS = _lib.CONSTANTS['ROMC_NM_INTS']
ROMC_NM_DONE = _lib.CONSTANTS['ROMC_NM_DONE']


def romc_nm_doubles(p):
    """Doubles of device Nelder-Mead state per problem (include/elfi_b200.h)."""
    return (p + 1) * (p + 1) + 3 * p + 2


def _romc_p(p):
    p = int(p)
    if not 1 <= p <= ROMC_MAX_P:
        raise ValueError('ROMC takes 1 <= p <= {} parameters, got {}'.format(ROMC_MAX_P, p))
    return p


def _dev_f64(x):
    t = x if dev.is_device_array(x) and x.dtype == torch.float64 else dev.to_device(x)
    return t.contiguous()


class RomcNelderMead:
    """P Nelder-Mead problems advanced in lock-step on the device (scipy's _minimize_neldermead
    with adaptive=False and no bounds).  ``theta`` (P, p) holds the point every problem needs
    next; pass f at those points to :meth:`step` until :meth:`running` is 0."""

    def __init__(self, x0, maxiter=None, maxfev=None, xatol=1e-4, fatol=1e-4):
        x0 = _dev_f64(x0)
        if x0.dim() != 2:
            raise ValueError('x0 must be (P, p), got shape {}'.format(tuple(x0.shape)))
        self.P, self.p = int(x0.shape[0]), _romc_p(x0.shape[1])
        self.maxiter = 200 * self.p if maxiter is None else int(maxiter)
        self.maxfev = 200 * self.p if maxfev is None else int(maxfev)
        if self.maxiter < 1 or self.maxfev < 1:
            raise ValueError('maxiter and maxfev must be positive')
        self.xatol, self.fatol = float(xatol), float(fatol)
        self.state = dev.empty((self.P, romc_nm_doubles(self.p)))
        self.istate = dev.empty((self.P, ROMC_NM_INTS), dtype=torch.int32)
        self.theta = dev.empty((self.P, self.p))
        _lib.call('elfi_b200_romc_nm_init_f64', dev.context(), self.P, self.p, dev.ptr(x0), self.p,
                  dev.ptr(self.state), dev.ptr(self.istate), dev.ptr(self.theta), self.p,
                  dev.stream_ptr())

    def step(self, fvals):
        f = _dev_f64(fvals).reshape(-1)
        if f.numel() != self.P:
            raise ValueError('step takes {} values, got {}'.format(self.P, f.numel()))
        _lib.call('elfi_b200_romc_nm_step_f64', dev.context(), self.P, self.p, dev.ptr(self.state),
                  dev.ptr(self.istate), dev.ptr(f), dev.ptr(self.theta), self.p, self.maxiter,
                  self.maxfev, self.xatol, self.fatol, dev.stream_ptr())

    def running(self):
        """Problems not finished (one device-to-host read)."""
        return int((self.istate[:, 0] != ROMC_NM_DONE).sum())

    def result(self):
        """Host (x_min (P, p), f_min (P,), nit (P,), nfev (P,), success (P,))."""
        s, i = dev.to_host(self.state), dev.to_host(self.istate)
        return (s[:, :self.p].copy(), s[:, -1].copy(), i[:, 1].astype(np.int64),
                i[:, 2].astype(np.int64), i[:, 4] == 0)


class RomcLineSearch:
    """romc.py line_search for the 2p (direction, side) pairs of every active problem in
    lock-step.  ``theta`` (2p, P, p) holds the next points; pass f at them, (2p, P), to
    :meth:`step` until :meth:`running` is 0.  ``limits()`` is the (P, p, 2) box of each problem."""

    def __init__(self, x_min, rot, active, eps, K=10, eta=1.0, rep_lim=300):
        self.x_min = _dev_f64(x_min)
        self.P, self.p = int(self.x_min.shape[0]), _romc_p(self.x_min.shape[1])
        self.rot = _dev_f64(rot)
        if tuple(self.rot.shape) != (self.P, self.p, self.p):
            raise ValueError('rot must be ({0}, {1}, {1})'.format(self.P, self.p))
        act = np.asarray(dev.to_host(active) if dev.is_device_array(active) else active).reshape(-1)
        if act.size != self.P:
            raise ValueError('active has {} entries, x_min {} rows'.format(act.size, self.P))
        self.active = dev.to_device(act.astype(np.int32), dtype=torch.int32)
        self.eps, self.K, self.eta, self.rep_lim = float(eps), int(K), float(eta), int(rep_lim)
        if self.K < 1 or self.rep_lim < 0 or not (self.eta > 0 and np.isfinite(self.eta)):
            raise ValueError('line search needs K >= 1, rep_lim >= 0 and a finite eta > 0')
        n = 2 * self.p * self.P
        self.state = dev.empty((n, self.p + 2))
        self.istate = dev.empty((n, 4), dtype=torch.int32)
        self.theta = dev.empty((2 * self.p, self.P, self.p))
        self._limits = dev.zeros((self.P, self.p, 2))
        self._call(1, None)

    def _call(self, init, f):
        _lib.call('elfi_b200_romc_line_search_f64', dev.context(), init, self.P, self.p,
                  dev.ptr(self.x_min), dev.ptr(self.rot), dev.ptr(self.active), dev.ptr(self.state),
                  dev.ptr(self.istate), dev.ptr(f), dev.ptr(self.theta), self.eps, self.K,
                  self.eta, self.rep_lim, dev.ptr(self._limits), dev.stream_ptr())

    def step(self, fvals):
        f = _dev_f64(fvals)
        if f.numel() != 2 * self.p * self.P:
            raise ValueError('step takes (2p, P) = ({}, {}) values'.format(2 * self.p, self.P))
        self._call(0, f)

    def running(self):
        return int((self.istate[:, 2] == 0).sum())

    def limits(self):
        return dev.to_host(self._limits)


def romc_box_sample(center, rot, rot_inv, limits, volume, n2, seed, coef=None):
    """n2 uniform draws from each of R rotated boxes (include/elfi_b200.h).  Returns device
    (pts (R, n2, p), q (R, n2), surr (R, n2) or None): q = contains / volume, surr the region's
    local quadratic (coef (R, 1 + p + p (p + 1) / 2)) at each point."""
    center = _dev_f64(center)
    R, p = int(center.shape[0]), _romc_p(center.shape[1])
    rot, rot_inv, limits, volume = (_dev_f64(a) for a in (rot, rot_inv, limits, volume))
    if tuple(rot.shape) != (R, p, p) or tuple(rot_inv.shape) != (R, p, p) or \
            tuple(limits.shape) != (R, p, 2) or volume.numel() != R:
        raise ValueError('box_sample takes center (R, p), rot and rot_inv (R, p, p), limits '
                         '(R, p, 2) and volume (R,)')
    n2 = int(n2)
    if n2 < 0:
        raise ValueError('n2 must be non-negative, got {}'.format(n2))
    if coef is not None:
        coef = _dev_f64(coef)
        if tuple(coef.shape) != (R, 1 + p + p * (p + 1) // 2):
            raise ValueError('coef must be (R, 1 + p + p (p + 1) / 2)')
    pts, q = dev.empty((R, n2, p)), dev.empty((R, n2))
    surr = None if coef is None else dev.empty((R, n2))
    _lib.call('elfi_b200_romc_box_sample_f64', dev.context(), R, p, n2, dev.ptr(center),
              dev.ptr(rot), dev.ptr(rot_inv), dev.ptr(limits), dev.ptr(volume),
              int(seed) & 0xffffffffffffffff, dev.ptr(coef), dev.ptr(pts), dev.ptr(q),
              dev.ptr(surr), dev.stream_ptr())
    return pts, q, surr


def romc_weights(dist, prior, q, eps):
    """(dist < eps) prior / q, 0 where q <= 0, elementwise; a device array of dist's shape."""
    dist, prior, q = (_dev_f64(a) for a in (dist, prior, q))
    n = dist.numel()
    if prior.numel() != n or q.numel() != n:
        raise ValueError('dist, prior and q must have the same number of entries')
    w = dev.empty(tuple(dist.shape))
    _lib.call('elfi_b200_romc_weights_f64', dev.context(), n, dev.ptr(dist), dev.ptr(prior),
              dev.ptr(q), float(eps), dev.ptr(w), dev.stream_ptr())
    return w


def romc_posterior_unnorm(theta, prior, eps, center=None, rot_inv=None, limits=None, coef=None,
                          fvals=None):
    """prior (M,) times the number of regions that count theta (M, p): with local models those
    containing it whose quadratic is <= eps, else those whose objective value fvals (M, R) is
    <= eps.  A device array (M,)."""
    theta = _dev_f64(theta)
    M, p = int(theta.shape[0]), _romc_p(theta.shape[1])
    prior = _dev_f64(prior)
    if prior.numel() != M:
        raise ValueError('prior has {} values, theta {} rows'.format(prior.numel(), M))
    if fvals is not None:
        fvals = _dev_f64(fvals)
        if fvals.dim() != 2 or int(fvals.shape[0]) != M:
            raise ValueError('fvals must be (M, R)')
        R = int(fvals.shape[1])
    else:
        center, rot_inv, limits, coef = (_dev_f64(a) for a in (center, rot_inv, limits, coef))
        R = int(center.shape[0])
        if tuple(center.shape) != (R, p) or tuple(rot_inv.shape) != (R, p, p) or \
                tuple(limits.shape) != (R, p, 2) or tuple(coef.shape) != (R, 1 + p + p * (p + 1) // 2):
            raise ValueError('posterior_unnorm takes center (R, p), rot_inv (R, p, p), limits '
                             '(R, p, 2) and coef (R, 1 + p + p (p + 1) / 2)')
    out = dev.empty((M,))
    _lib.call('elfi_b200_romc_posterior_unnorm_f64', dev.context(), M, R, p, dev.ptr(theta), p,
              dev.ptr(center), dev.ptr(rot_inv), dev.ptr(limits), dev.ptr(coef), dev.ptr(fvals),
              R, float(eps), dev.ptr(prior), dev.ptr(out), dev.stream_ptr())
    return out


# ---- regression adjustment (elfi/methods/post_processing.py: LinearAdjustment) ----------------------
REGADJ_D_MAX = _lib.CONSTANTS['REGADJ_D_MAX']
REGADJ_N_MAX = _lib.CONSTANTS['REGADJ_N_MAX']


def _regadj_shape(x):
    return tuple(x.shape) if hasattr(x, 'shape') else np.shape(x)


def _regadj_block(X, name):
    """X as an (N, w) float64 device matrix with unit column stride: an (N, w) array, or a list of w
    (N,) columns (stacked here).  Shapes are checked before anything is uploaded."""
    if isinstance(X, (list, tuple)):
        if not X:
            raise ValueError('{} has no columns'.format(name))
        lengths = set()
        for j, c in enumerate(X):
            shape = _regadj_shape(c)
            if len(shape) != 1:
                raise ValueError('{} column {} must be 1-d (one scalar per row), got shape {}'.format(
                    name, j, shape))
            lengths.add(shape[0])
        if len(lengths) != 1:
            raise ValueError('the columns of {} differ in length: {}'.format(name, sorted(lengths)))
        N = lengths.pop()
        if N > REGADJ_N_MAX:
            raise ValueError('{} has N = {} rows; linear_adjust takes N < 2^31'.format(name, N))
        cols = [c if dev.is_device_array(c) and c.dtype == torch.float64 else dev.to_device(c)
                for c in X]
        return torch.stack(cols, dim=1)
    shape = _regadj_shape(X)
    if len(shape) != 2:
        raise ValueError('{} must be an (N, width) array or a list of (N,) columns, got shape '
                         '{}'.format(name, shape))
    if shape[0] > REGADJ_N_MAX:
        raise ValueError('{} has N = {} rows; linear_adjust takes N < 2^31'.format(name, shape[0]))
    M = X if dev.is_device_array(X) and X.dtype == torch.float64 else dev.to_device(X)
    if M.shape[0] > 0 and (M.stride(1) != 1 or M.stride(0) < M.shape[1]):
        M = M.contiguous()
    return M


def _regadj_solve(M, q, n, tol):
    """The minimum-norm least-squares coefficients of the centred normal equations: the q x q block
    A = X_c^T X_c and the q x pg block B = X_c^T Y_c of M.  Eigenvalues lambda <= tol^2 lambda_max
    count as zero (scikit-learn's singular-value cut sigma <= tol sigma_max on X_c).  Returns coef
    (q, pg), the rank and the singular values of X_c (descending, min(n, q) of them)."""
    A, B = M[:q, :q], M[:q, q:]
    w, V = np.linalg.eigh(A)
    keep = w > tol * tol * w[-1] if w[-1] > 0 else np.zeros(q, dtype=bool)
    Vr = V[:, keep]
    coef = Vr @ ((Vr.T @ B) / w[keep][:, None])
    singular = np.sqrt(np.clip(w[::-1], 0.0, None))[:min(n, q)]
    return coef, int(keep.sum()), singular


def linear_adjust(S, theta, observed, tol=1e-6):
    """The local-linear regression adjustment of Beaumont et al. (2002), one least-squares fit with
    an intercept per parameter, regressors x_i = S_i - observed.

    S is (N, q) and theta (N, p), host or device, each as an array (any row stride) or a list of
    (N,) columns.  Parameter k is fitted on the rows whose summaries and theta_k are finite; every
    parameter without a non-finite theta_k on such rows shares one fit.  Each fit reads back its
    count, means and centred (q + p_g)^2 moments and solves them on the host (_regadj_solve).

    Returns (adjusted, fits): adjusted[k] is a device column (n_k,) of theta_k - x @ coef_k over
    parameter k's rows in row order; fits[k] is a dict with 'coef' (q,), 'intercept', 'rank',
    'singular' and 'n_rows'.  ValueError for q + p > REGADJ_D_MAX, N >= 2^31, a column that is not
    1-d, or a parameter without any finite row."""
    tol = float(tol)
    if not tol >= 0:
        raise ValueError('tol must be non-negative, got {}'.format(tol))
    Sd = _regadj_block(S, 'S')
    Td = _regadj_block(theta, 'theta')
    N, q = int(Sd.shape[0]), int(Sd.shape[1])
    p = int(Td.shape[1])
    if int(Td.shape[0]) != N:
        raise ValueError('S has {} rows, theta {}'.format(N, int(Td.shape[0])))
    if q < 1 or p < 1 or q + p > REGADJ_D_MAX:
        raise ValueError('linear_adjust takes q >= 1 summaries and p >= 1 parameters with q + p <= '
                         '{}, got q = {}, p = {}'.format(REGADJ_D_MAX, q, p))
    if N == 0:
        raise ValueError('linear_adjust needs at least one row, got N = 0')
    o = dev.to_device(observed).reshape(-1).contiguous()
    if o.numel() != q:
        raise ValueError('observed has {} values, S has q = {} summaries'.format(o.numel(), q))
    ctx, stream = dev.context(), dev.stream_ptr()
    shape = (dev.ptr(Sd), _ld(Sd), N, q, dev.ptr(o), dev.ptr(Td), _ld(Td), p)
    flags = dev.empty((N,), dtype=torch.uint8)
    counts = dev.empty((p + 1,), dtype=torch.int64)
    _lib.call('elfi_b200_regadj_mask_f64', ctx, *shape, dev.ptr(flags), dev.ptr(counts), stream)
    bad = dev.to_host(counts)[1:]
    shared = [k for k in range(p) if bad[k] == 0]
    groups = ([(shared, -1)] if shared else []) + [([k], k) for k in range(p) if bad[k] != 0]
    adjusted, fits = [None] * p, [None] * p
    for cols, sel in groups:
        pg = len(cols)
        d = q + pg
        cols_h = np.ascontiguousarray(cols, dtype=np.int32)
        mom = dev.empty((1 + d + d * d,))
        _lib.call('elfi_b200_regadj_moments_f64', ctx, *shape, dev.ptr(flags),
                  ctypes.c_void_p(cols_h.ctypes.data), pg, sel, dev.ptr(mom), stream)
        h = dev.to_host(mom)
        n = int(h[0])
        if n == 0:
            raise ValueError('no row has finite summaries and a finite value of parameter {}: '
                             'nothing to fit (n_samples = 0)'.format(cols[0]))
        mean, M = h[1:1 + d], h[1 + d:].reshape(d, d)
        coef, rank, singular = _regadj_solve(M, q, n, tol)
        intercept = mean[q:] - mean[:q] @ coef
        coef_d = dev.to_device(np.ascontiguousarray(coef))
        out = dev.empty((pg, n))
        _lib.call('elfi_b200_regadj_adjust_f64', ctx, *shape, dev.ptr(flags),
                  ctypes.c_void_p(cols_h.ctypes.data), pg, sel, int(sel < 0 and n == N),
                  dev.ptr(coef_d), dev.ptr(out), n, stream)
        for kk, k in enumerate(cols):
            adjusted[k] = out[kk]
            fits[k] = dict(coef=coef[:, kk].copy(), intercept=float(intercept[kk]), rank=rank,
                           singular=singular.copy(), n_rows=n)
    return adjusted, fits


# ---- user-written simulators, compiled at run time (csrc/usersim.cu, csrc/usersim_rt.cuh) ---------
USERSIM_P_MAX = _lib.CONSTANTS['USERSIM_P_MAX']
USERSIM_N_OUT_MAX = _lib.CONSTANTS['USERSIM_N_OUT_MAX']
USERSIM_N_SUM_MAX = _lib.CONSTANTS['USERSIM_N_SUM_MAX']
USERSIM_LOCAL_MAX = _lib.CONSTANTS['USERSIM_LOCAL_MAX']
_USERSIM_LOG_CHARS = 1 << 16
_usersim_refs = {}        # (device, handle address) -> references taken by usersim_compile
_usersim_compiled = [0]   # NVRTC compilations run by usersim_compile


class UserSimulator:
    """A simulator compiled by :func:`usersim_compile` for one device: its library handle and the
    shapes it was compiled for."""

    def __init__(self, handle, device, n_params, n_out, n_summaries, salt):
        self.handle = handle
        self.device = device
        self.n_params = n_params
        self.n_out = n_out
        self.n_summaries = n_summaries
        self.salt = salt


def _count(value, lo, hi, what):
    if isinstance(value, (bool, np.bool_)) or int(value) != value or not lo <= value <= hi:
        raise ValueError('a user simulator takes an integer {} <= {} <= {}, got {!r}'.format(
            lo, what, hi, value))
    return int(value)


def usersim_shapes(n_params, n_out, n_summaries=0, salt=0):
    """(n_params, n_out, n_summaries, salt) as ints, or ValueError when one is out of the range
    elfi_b200.h gives it."""
    return (_count(n_params, 1, USERSIM_P_MAX, 'n_params'),
            _count(n_out, 1, USERSIM_N_OUT_MAX, 'n_out'),
            _count(n_summaries, 0, USERSIM_N_SUM_MAX, 'n_summaries'),
            _count(salt, 0, 2 ** 32 - 1, 'salt'))


def usersim_compile(source, n_params, n_out, n_summaries=0, salt=0):
    """Compile a user's CUDA simulator for the current device (NVRTC, sm_90a) and load it.

    ``source`` defines ``__device__ void simulate(const double* theta, elfi::RowStream& rng,
    double* y)``, which writes the n_out values of one row from its n_params parameters, and, when
    n_summaries > 0, ``__device__ void summarise(const double* y, double* s)``, which writes a
    row's n_summaries summaries; elfi_b200/csrc/usersim_rt.cuh states the contract.  ``salt`` is
    the fourth counter word of the simulator's Philox blocks.  The context caches compiled sources:
    the same (source, shapes, salt) again returns the same simulator without running NVRTC.

    Returns a :class:`UserSimulator`.  Shapes are checked before anything is compiled (ValueError);
    a source NVRTC refuses raises ElfiB200Error carrying NVRTC's log, whose line numbers are the
    source's own."""
    if not isinstance(source, str) or not source.strip():
        raise ValueError('the simulator source must be a non-empty string')
    n_params, n_out, n_summaries, salt = usersim_shapes(n_params, n_out, n_summaries, salt)
    ctx = dev.context()
    device = dev.current_device()
    log = ctypes.create_string_buffer(_USERSIM_LOG_CHARS)
    handle = ctypes.c_void_p()
    try:
        _lib.call('elfi_b200_usersim_compile', ctx, source.encode('utf-8'), n_params, n_out,
                  n_summaries, salt, log, len(log), ctypes.byref(handle))
    except _lib.ElfiB200Error as e:
        text = log.value.decode('utf-8', 'replace')
        if not text:
            raise
        hint = ''
        if 'Unresolved extern function' in text:
            hint = ('\nThe source must define __device__ void simulate(const double* theta, '
                    'elfi::RowStream& rng, double* y){}.'.format(
                        ' and __device__ void summarise(const double* y, double* s)'
                        if n_summaries else ''))
        raise _lib.ElfiB200Error('NVRTC could not compile the user simulator:\n{}{}'.format(
            text, hint)) from e
    key = (device, handle.value)
    if key not in _usersim_refs:
        _usersim_compiled[0] += 1
    _usersim_refs[key] = _usersim_refs.get(key, 0) + 1
    return UserSimulator(handle, device, n_params, n_out, n_summaries, salt)


def usersim_compiles():
    """How many times :func:`usersim_compile` has run NVRTC in this process (cache hits do not
    count)."""
    return _usersim_compiled[0]


def usersim_release(sim):
    """Give back the reference :func:`usersim_compile` took; the last one frees the simulator."""
    key = (sim.device, sim.handle.value)
    if _usersim_refs.get(key, 0) <= 0:
        raise ValueError('this user simulator has been released already')
    _lib.call('elfi_b200_usersim_release', dev.context(sim.device), sim.handle)
    _usersim_refs[key] -= 1
    if _usersim_refs[key] == 0:
        del _usersim_refs[key]
        sim.handle = ctypes.c_void_p()


def _usersim_ctx(sim):
    if (sim.device, sim.handle.value) not in _usersim_refs:
        raise ValueError('this user simulator has been released')
    if dev.current_device() != sim.device:
        raise ValueError('the user simulator was compiled for cuda:{}, the current device is '
                         'cuda:{}'.format(sim.device, dev.current_device()))
    return dev.context(sim.device)


def usersim_run(sim, params, seed=0, offset=0, want_data=False, want_summaries=True):
    """Run a :class:`UserSimulator` on a batch: row i has parameters ``params[j][i]`` (n_params
    columns of one length, device or host; or one (batch, n_params) matrix) and is row offset + i
    of the Philox stream keyed by ``seed``, so a row does not depend on how a batch is split.

    Returns (Y, S), each None unless asked for: Y (batch, n_out) the data and S (batch,
    n_summaries) the summaries.  Summaries without the data are computed in the simulator's
    kernel without writing the data when n_out <= USERSIM_LOCAL_MAX, bit for bit the summaries of
    a run that writes it."""
    if not (want_data or want_summaries):
        raise ValueError('usersim_run asked for neither the data nor the summaries')
    if want_summaries and sim.n_summaries == 0:
        raise ValueError('the user simulator has no summaries (n_summaries = 0)')
    if isinstance(params, (list, tuple)):
        cols = [dev.to_device(c).reshape(-1).contiguous() for c in params]
    else:
        P = _matrix(params)
        cols = [P[:, j].contiguous() for j in range(P.shape[1])]
    if len(cols) != sim.n_params:
        raise ValueError('the user simulator takes {} parameters, got {}'.format(
            sim.n_params, len(cols)))
    B = int(cols[0].numel())
    if any(int(c.numel()) != B for c in cols):
        raise ValueError('the parameter columns must have one length, got {}'.format(
            [int(c.numel()) for c in cols]))
    ctx = _usersim_ctx(sim)
    fused = want_summaries and not want_data and sim.n_out <= USERSIM_LOCAL_MAX
    Y = None if fused else dev.empty((B, sim.n_out))
    S = dev.empty((B, sim.n_summaries)) if want_summaries else None
    mode = 2 if fused else (1 if want_summaries else 0)
    ptrs = (ctypes.c_void_p * len(cols))(*[c.data_ptr() for c in cols])
    _lib.call('elfi_b200_usersim_launch', ctx, sim.handle, ptrs, B, int(seed), int(offset), mode,
              dev.ptr(Y), sim.n_out, dev.ptr(S), max(1, sim.n_summaries), dev.stream_ptr())
    return (Y if want_data else None), S


def usersim_summarise(sim, y):
    """The summaries a :class:`UserSimulator`'s ``summarise`` gives the rows of y (batch, n_out)
    or the one row y (n_out,): observed data, say, or data kept in a sample.  Returns S (batch,
    n_summaries)."""
    y = y if dev.is_device_array(y) else np.asarray(y, dtype=np.float64)
    if sim.n_summaries == 0:
        raise ValueError('the user simulator has no summaries (n_summaries = 0)')
    Y = _matrix(y.reshape(1, -1) if y.ndim == 1 else y)
    if Y.shape[1] != sim.n_out:
        raise ValueError('the user simulator summarises rows of {} values, got shape {}'.format(
            sim.n_out, tuple(Y.shape)))
    B = int(Y.shape[0])
    ctx = _usersim_ctx(sim)
    S = dev.empty((B, sim.n_summaries))
    ptrs = (ctypes.c_void_p * 1)()
    _lib.call('elfi_b200_usersim_launch', ctx, sim.handle, ptrs, B, 0, 0, 3, dev.ptr(Y),
              _ld(Y), dev.ptr(S), sim.n_summaries, dev.stream_ptr())
    return S
