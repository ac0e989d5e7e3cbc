"""Bodies of the tests of the resident rejection step (shared by the CPU-double and GPU
collections): CandidateBuffer.bind_batch -> elfi_b200_rejection_batch_f64 (distances, acceptance,
mask compaction, append of [d | extras] and the device-side counts) followed by
CandidateBuffer.best, checked bit for bit against the C oracle's distances and acceptance
(elfi_oracle.cdist_euclid / nested_distance / accept_indices, bit-exact to SciPy's cdist) and the
reference's merge (samplers.py:209-237, restated as merge_cases.reference_merge).

The step does no arithmetic beyond the distances, so every comparison is exact: np.array_equal on
float64 values, NaN-aware where NaN is expected.  After every batch a case checks d_out,
acc_idx[:n_acc] and n_acc; at the end count, dropped, every packed row of the buffer (rows at or
beyond count keep the NaN the buffer was filled with) and best(n)."""
import contextlib
import ctypes

import numpy as np
import torch

import elfi_oracle as o
from merge_cases import reference_merge

# ---------------------------------------------------------------------------- shape tables
# (D, ld) of the two distance paths of launch_dist: the TMA row stream needs D >= 16 and a 16-byte
# aligned leading dimension; narrower matrices and odd leading dimensions take the direct kernel
ROWSTREAM = [(24, 24), (128, 128), (256, 256)]
DIRECT = [(2, 2), (15, 15), (21, 33)]
# batch sizes across a warp's 32-row mask word and compact_mask_kernel's CTA (1024 mask words,
# 32768 rows), up to several CTAs
SIZES = [1, 31, 32, 33, 32767, 32768, 32769, 65537, 100003]
# every size on both paths, each (D, ld) at three sizes
SHAPES = [(path, D, ld, B) for i, B in enumerate(SIZES)
          for path, (D, ld) in (('rowstream', ROWSTREAM[i % 3]), ('direct', DIRECT[(i + 1) % 3]))]
LARGEST = max(SHAPES, key=lambda s: s[3] * s[1])

# every NestedConsumer<KMAX> instance (2, 3, 4, 5, 6, 8, 16, 32) and K < KMAX inside one (7, 17);
# K = 1 is the weighted single column
NESTED_K = [1, 2, 3, 4, 5, 6, 7, 16, 17, 32]
# (width, layout) of up to 7 extra sources: 8 sources with d, the most one append takes
EXTRA_LAYOUTS = [(1, 'contig'), (2, 'view'), (5, 'contig'), (1, 'strided'), (2, 'contig'),
                 (5, 'view'), (1, 'view')]
N_EXTRA = [0, 1, 3, 7]
CAPACITY_KINDS = ['exact', 'first_batch', 'third_batch', 'zero', 'reset']
THRESHOLD_KINDS = ['host_sequence', 'device', 'device_updated', 'equal', 'inf', 'minus_one',
                   'nan', 'nonfinite_rows', 'nonfinite_rows_inf']
RAW_KINDS = ['null_idx', 'null_dropped', 'wide_dst', 'max_rows_zero']


def _host(t):
    return t.cpu().numpy()


def _cols(a, B):
    return np.asarray(a, dtype=np.float64).reshape(B, -1)


# ------------------------------------------------------------------------------ the reference
def oracle_distances(S, obs, v=None):
    """(B, K) distances: cdist(S, obs) without weights, else the reference's nested distance with
    cdist weights v[k] ** 2 (elfi_model.py:1135-1151)."""
    if v is None:
        return o.cdist_euclid(S, obs).reshape(-1, 1)
    return o.nested_distance(S, obs, list(v))


class Expected:
    """The candidate buffer the step must leave: the accepted rows [d | extras] of each batch in
    acc_idx order behind the count, until the capacity runs out; the rest counted as dropped."""

    def __init__(self, capacity, width):
        self.capacity = capacity
        self.rows = np.full((capacity, width), np.nan)
        self.count = self.dropped = 0
        self.batches = []      # for reference_merge: {'d': (B, K), 'e0': ..., ...}

    def add(self, d, extras, thr):
        B = d.shape[0]
        idx = o.accept_indices(d, thr)
        packed = np.column_stack([d] + [_cols(e, B) for e in extras])
        keep = idx[:max(0, self.capacity - self.count)]
        self.rows[self.count:self.count + len(keep)] = packed[keep]
        self.count += len(keep)
        self.dropped += len(idx) - len(keep)
        self.batches.append(dict({'d': d}, **{'e{}'.format(i): e for i, e in enumerate(extras)}))
        return idx

    def best(self, n, key):
        """The project's best-n: the kept rows ranked by `key`, ties in append order."""
        kept = self.rows[:self.count]
        return kept[np.argsort(kept[:, key], kind='stable')[:n]]

    def merged(self, thr, n, pad=np.inf):
        """The reference's merge of the same batches, packed as buffer rows (first min(n, count))."""
        want = reference_merge(self.batches, thr, n, pad)
        names = ['d'] + ['e{}'.format(i) for i in range(len(self.batches[0]) - 1)]
        packed = np.column_stack([want[k] if want[k].ndim == 2 else want[k][:, None]
                                  for k in names])
        return packed[:min(n, self.count)]


# ------------------------------------------------------------------------- device inputs
class Source:
    """A device array of B rows in one of the layouts a caller hands the step, refilled in place
    before each batch (the bound call keeps its pointer).  The storage around the view holds NaN,
    so a read from the wrong columns shows."""

    def __init__(self, B, width, layout):
        from elfi_b200 import device as dev
        self.width = width
        if layout == 'contig':
            self.storage = dev.full((B, width), np.nan)
            self.view = self.storage[:, 0] if width == 1 else self.storage
        elif layout == 'view':                # columns of a wider matrix: ld > width
            self.storage = dev.full((B, width + 3), np.nan)
            self.view = self.storage[:, 2:2 + width]
        elif layout == 'strided':             # a 1-d column of a wider matrix
            assert width == 1
            self.storage = dev.full((B, 3), np.nan)
            self.view = self.storage[:, 1]
        else:
            raise ValueError(layout)

    def fill(self, host):
        from elfi_b200 import device as dev
        self.view.copy_(dev.to_device(np.asarray(host).reshape(self.view.shape)))


class Step:
    """One bound rejection step: S (B, D) with leading dimension ld, the observed row, optional
    nested weights (K, D), extras in the given (width, layout)s, a candidate buffer of `capacity`
    rows filled with NaN, and thresholds on the host (fixed at binding) or in a device tensor that
    is refilled before each batch."""

    def __init__(self, B, D, ld, obs, capacity, thr, W=None, layouts=(), thr_mode='device',
                 buf=None):
        from elfi_b200 import device as dev
        from elfi_b200 import ops
        self.B, self.D = B, D
        self.K = 1 if W is None else W.shape[0]
        self.S_store = dev.full((B, ld), np.nan)
        self.S = self.S_store[:, :D]
        self.extras = [Source(B, w, lay) for w, lay in layouts]
        widths = [self.K] + [w for w, _ in layouts]
        self.buf = buf if buf is not None else ops.CandidateBuffer(capacity, widths)
        self.buf.rows.fill_(np.nan)
        self.d_out = dev.empty((B,) if self.K == 1 else (B, self.K))
        self.acc_idx = dev.empty((B,), dtype=torch.int32)
        self.n_acc = dev.zeros((1,), dtype=torch.int64)
        self.thr_dev = None
        if thr_mode == 'device':
            self.thr_dev = dev.to_device(np.atleast_1d(thr))
            thresholds = self.thr_dev
        elif thr_mode == 'host':
            thresholds = np.atleast_1d(np.asarray(thr, dtype=np.float64)).copy()
        else:                                  # a plain Python sequence
            thresholds = [float(t) for t in np.atleast_1d(thr)]
        self.run = self.buf.bind_batch(self.S, dev.to_device(obs), thresholds, self.d_out,
                                       self.acc_idx, self.n_acc, [e.view for e in self.extras],
                                       w=W)

    def batch(self, S, extras, thr=None):
        """Refill the inputs (and the device thresholds), run the bound step, return
        (d_out (B, K), accepted indices, n_acc) as host arrays."""
        from elfi_b200 import device as dev
        self.S.copy_(dev.to_device(S))
        for src, host in zip(self.extras, extras):
            src.fill(host)
        if thr is not None:
            self.thr_dev.copy_(dev.to_device(np.atleast_1d(thr)))
        self.run()
        n = int(self.n_acc.item())
        return _host(self.d_out).reshape(self.B, self.K), _host(self.acc_idx)[:n], n


def run_batches(step, exp, batches, thrs, obs, v=None):
    """Each (S, extras) batch through the bound step against the oracle, with the thresholds
    thrs[i] in force (pushed to the device tensor when the step reads one)."""
    for (S, extras), thr in zip(batches, thrs):
        d, idx, n = step.batch(S, extras, thr if step.thr_dev is not None else None)
        want_d = oracle_distances(S, obs, v)
        want_idx = exp.add(want_d, extras, thr)
        assert np.array_equal(d, want_d, equal_nan=True), 'd_out differs from the oracle'
        assert n == len(want_idx), ('n_acc', n, len(want_idx))
        assert np.array_equal(idx, want_idx), 'acc_idx differs from accept_indices'


def check_buffer(step, exp):
    """count, dropped and every row of the buffer, the unfilled ones still NaN."""
    buf = step.buf
    assert int(buf.count.item()) == exp.count, ('count', int(buf.count.item()), exp.count)
    assert int(buf.dropped.item()) == exp.dropped, ('dropped', int(buf.dropped.item()),
                                                    exp.dropped)
    assert np.array_equal(_host(buf.rows), exp.rows, equal_nan=True), 'packed rows differ'


def check_best(step, exp, ns, thr=None, pad=np.inf):
    """best(n) for every n in ns against the project's order and, when the thresholds stayed fixed
    and nothing was dropped (`thr` given), against the reference's merge.  The default key is the
    reference's: the last distance column."""
    key = step.K - 1
    for n in ns:
        top, count, dropped = step.buf.best(n)
        top = _host(top)
        assert (count, dropped) == (exp.count, exp.dropped)
        want = exp.best(n, key)
        assert top.shape == want.shape and np.array_equal(top, want), ('best', n)
        if thr is not None:
            assert exp.dropped == 0
            assert np.array_equal(top, exp.merged(thr, n, pad)), ('reference merge', n)
        if step.K > 1:
            keyed, _, _ = step.buf.best(n, key_col=key)
            assert np.array_equal(_host(keyed), top)


def _batches(rs, nb, B, D, layouts, dup=None):
    """nb host batches (S, [extras]); dup maps a batch to an earlier one whose S it repeats."""
    out = []
    for i in range(nb):
        S = rs.randn(B, D)
        if dup and i in dup:
            S = out[dup[i]][0].copy()
        out.append((S, [rs.randn(B, w) if w > 1 else rs.randn(B) for w, _ in layouts]))
    return out


def _obs(rs, D):
    return 0.3 * rs.randn(D)


# ---------------------------------------------------------------------------------- the cases
def case_path_shape(path, D, ld, B):
    """Three batches of B rows through one distance path, K = 1 and two width-1 extras, host
    thresholds; no row is dropped, so best(n) is the reference's merge."""
    rs = np.random.RandomState(B * 7 + D)
    obs = _obs(rs, D)
    layouts = [(1, 'contig'), (1, 'strided')]
    batches = _batches(rs, 3, B, D, layouts)
    thr = float(np.quantile(oracle_distances(batches[0][0], obs), 0.3))
    step = Step(B, D, ld, obs, 3 * B + 1, thr, layouts=layouts, thr_mode='host')
    exp = Expected(3 * B + 1, 3)
    run_batches(step, exp, batches, [thr] * 3, obs)
    check_buffer(step, exp)
    n = max(1, exp.count // 3)
    check_best(step, exp, [n, exp.count], thr=thr)
    return step, exp


def _nested_weights(rs, K, D):
    v = 0.5 + rs.rand(K, D)                 # the reference's scale ** -1 (cdist w = v ** 2)
    return v, v ** 2


def case_nested(K, path):
    """K nested weighted distances through the append: a row is accepted when all K columns are
    within their thresholds, and best(n) ranks by the last column, as the reference does."""
    D, ld = (24, 24) if path == 'rowstream' else (15, 15)
    B = 3000
    rs = np.random.RandomState(100 + K)
    obs = _obs(rs, D)
    v, W = _nested_weights(rs, K, D)
    layouts = [(1, 'contig')]
    batches = _batches(rs, 3, B, D, layouts)
    d0 = oracle_distances(batches[0][0], obs, v)
    for q in (0.5, 0.7, 0.8, 0.9, 0.95, 0.98):    # every column binds, some rows pass all
        thr = np.quantile(d0, q, axis=0)
        if len(o.accept_indices(d0, thr)) >= B // 20:
            break
    step = Step(B, D, ld, obs, 3 * B, thr, W=W, layouts=layouts)
    exp = Expected(3 * B, K + 1)
    run_batches(step, exp, batches, [thr] * 3, obs, v)
    check_buffer(step, exp)
    if K > 1:
        # the case has teeth: the last column alone accepts more rows than all K together, and
        # the first column ranks the kept rows in another order than the last
        assert len(o.accept_indices(d0[:, -1:], thr[-1:])) > len(o.accept_indices(d0, thr)) > 0
        kept = exp.rows[:exp.count]
        assert not np.array_equal(np.argsort(kept[:, 0], kind='stable'),
                                  np.argsort(kept[:, K - 1], kind='stable'))
    check_best(step, exp, [50, exp.count], thr=thr)
    return step, exp


def case_default_key_is_reference_key():
    """best(n) without a key ranks nested distances by the reference's key, the last column
    (samplers.py:231-233), not by the first."""
    K, D, B, n = 3, 24, 2000, 200
    rs = np.random.RandomState(7)
    obs = _obs(rs, D)
    v, W = _nested_weights(rs, K, D)
    S = rs.randn(B, D)
    thr = np.full(K, np.inf)
    step = Step(B, D, D, obs, B, thr, W=W)
    step.batch(S, [], thr)
    want = reference_merge([{'d': oracle_distances(S, obs, v)}], thr, n)['d']
    top, _, _ = step.buf.best(n)
    assert np.array_equal(_host(top), want), 'best(n) does not rank by the last distance column'


def case_extras(n_extra):
    """n_extra extra sources of widths 1, 2 and 5, contiguous, as columns of a wider matrix and as
    a strided 1-d column: every packed column from its own source and row."""
    D, B = 24, 2000
    rs = np.random.RandomState(200 + n_extra)
    obs = _obs(rs, D)
    layouts = EXTRA_LAYOUTS[:n_extra]
    batches = _batches(rs, 3, B, D, layouts)
    thr = float(np.quantile(oracle_distances(batches[0][0], obs), 0.25))
    width = 1 + sum(w for w, _ in layouts)
    step = Step(B, D, D, obs, 3 * B, thr, layouts=layouts)
    exp = Expected(3 * B, width)
    run_batches(step, exp, batches, [thr] * 3, obs)
    check_buffer(step, exp)
    check_best(step, exp, [100, exp.count], thr=thr)


def case_capacity(kind):
    """The buffer runs out: exactly at the end, in the middle of the first batch, in the middle of
    batch 3 of 5 (batches 4 and 5 are dropped whole and `dropped` accumulates), capacity 0, and a
    reset() before the same buffer and binding run again."""
    D, B = 24, 4000
    rs = np.random.RandomState(300)
    obs = _obs(rs, D)
    layouts = [(1, 'contig'), (2, 'view')]
    batches = _batches(rs, 5, B, D, layouts)
    thr = float(np.quantile(oracle_distances(batches[0][0], obs), 0.2))
    acc = [len(o.accept_indices(oracle_distances(S, obs), thr)) for S, _ in batches]
    capacity = {'exact': sum(acc), 'first_batch': acc[0] // 2,
                'third_batch': acc[0] + acc[1] + acc[2] // 2, 'zero': 0,
                'reset': acc[0] + acc[1] // 3}[kind]
    step = Step(B, D, D, obs, capacity, thr, layouts=layouts)
    exp = Expected(capacity, 4)
    run_batches(step, exp, batches, [thr] * 5, obs)
    check_buffer(step, exp)
    if kind == 'exact':
        assert exp.dropped == 0 and exp.count == capacity
    elif kind == 'third_batch':
        assert exp.dropped == acc[2] - acc[2] // 2 + acc[3] + acc[4]
    elif kind == 'reset':
        step.buf.reset()
        step.buf.rows.fill_(np.nan)
        exp = Expected(capacity, 4)
        run_batches(step, exp, batches[1:], [thr] * 4, obs)
        check_buffer(step, exp)
    check_best(step, exp, [0, 1, exp.count], thr=thr if exp.dropped == 0 else None)


def case_thresholds(kind):
    """Thresholds from a host sequence or a device tensor, a device tensor updated in place between
    calls of one bound step (each batch is accepted against the threshold in force when it ran), a
    threshold equal to a distance (`<=` accepts it), +inf, -1 and NaN thresholds, and NaN / +inf
    rows of S (rejected by a finite threshold, +inf ones accepted by +inf; their distances still
    the oracle's)."""
    D, B = 24, 3000
    rs = np.random.RandomState(400)
    obs = _obs(rs, D)
    layouts = [(1, 'contig')]
    batches = _batches(rs, 4, B, D, layouts)
    if kind.startswith('nonfinite_rows'):
        for i, (S, _) in enumerate(batches):
            S[5 + i::97, 3] = np.nan
            S[11 + i::89, 7] = np.inf
            S[13 + i::101, :] = -np.inf
    d0 = oracle_distances(batches[0][0], obs)
    q = float(np.nanquantile(d0[np.isfinite(d0)], 0.3))
    thr = {'host_sequence': q, 'device': q, 'device_updated': q, 'inf': np.inf, 'minus_one': -1.0,
           'nan': np.nan, 'nonfinite_rows': q, 'nonfinite_rows_inf': np.inf}.get(kind)
    if kind == 'equal':
        thr = float(np.sort(d0[:, 0])[B // 4])
    thrs = [thr] * 4
    if kind == 'device_updated':
        thrs = [q, float(np.quantile(d0, 0.05)), np.inf, -1.0]
    mode = {'host_sequence': 'sequence', 'equal': 'host', 'minus_one': 'host'}.get(kind, 'device')
    step = Step(B, D, D, obs, 4 * B, thrs[0], layouts=layouts, thr_mode=mode)
    exp = Expected(4 * B, 2)
    run_batches(step, exp, batches, thrs, obs)
    check_buffer(step, exp)
    if kind == 'equal':
        assert np.any(exp.rows[:exp.count, 0] == thr), 'the tie with the threshold was not kept'
    if kind in ('minus_one', 'nan'):
        assert exp.count == 0
    if kind == 'inf':
        assert exp.count == 4 * B
    if kind.startswith('nonfinite_rows'):
        d_all = np.concatenate([oracle_distances(S, obs) for S, _ in batches])
        assert np.isnan(d_all).any() and np.isinf(d_all).any()
        n_inf = int(np.isinf(d_all).sum())
        assert np.isinf(exp.rows[:exp.count, 0]).sum() == (n_inf if thr == np.inf else 0)
        assert not np.isnan(exp.rows[:exp.count, 0]).any()
    fixed = kind != 'device_updated'
    check_best(step, exp, [0, 1, exp.count, exp.count + 5], thr=thr if fixed else None,
               pad=np.nan)


def case_best_ties():
    """best(n) for n = 0, 1, count and more than count, over batches that repeat earlier rows of S
    with other extras: exact ties, kept in append order."""
    D, B = 24, 1500
    rs = np.random.RandomState(500)
    obs = _obs(rs, D)
    layouts = [(1, 'contig'), (2, 'contig')]
    batches = _batches(rs, 4, B, D, layouts, dup={2: 0, 3: 0})
    thr = float(np.quantile(oracle_distances(batches[0][0], obs), 0.2))
    step = Step(B, D, D, obs, 4 * B, thr, layouts=layouts)
    exp = Expected(4 * B, 4)
    run_batches(step, exp, batches, [thr] * 4, obs)
    check_buffer(step, exp)
    check_best(step, exp, [0, 1, exp.count, exp.count + 7], thr=thr)
    # spelled out: each accepted row of batch 0 comes back three times in a row, with the
    # extras of batches 0, 2 and 3 in that order
    top = _host(step.buf.best(exp.count)[0])
    d0 = oracle_distances(batches[0][0], obs)[:, 0]
    idx0 = o.accept_indices(d0, thr)
    assert len(idx0) > 0
    for j in idx0[:50]:
        at = np.flatnonzero(top[:, 0] == d0[j])
        assert np.array_equal(at, at[0] + np.arange(3))
        assert np.array_equal(top[at, 1], [batches[i][1][0][j] for i in (0, 2, 3)])


def case_raw_append(kind):
    """elfi_b200_accept_append_f64 through _lib.call: acc_idx NULL (rows 0 .. n_acc), dropped
    NULL, ld_dst beyond the total width (the padding columns stay untouched), max_rows 0 (no
    launch, nothing changes)."""
    from elfi_b200 import _lib
    from elfi_b200 import device as dev
    rs = np.random.RandomState(600)
    B, widths = 40, [1, 3]
    srcs_h = [rs.randn(B, w) for w in widths]
    srcs = [dev.to_device(s) for s in srcs_h]
    width = sum(widths)
    ld_dst = width + 3 if kind == 'wide_dst' else width
    capacity = 25
    dst = dev.full((capacity, ld_dst), -7.5)
    count0, dropped0 = (3, 2) if kind == 'max_rows_zero' else (4, 1)
    count = dev.to_device(np.array([count0]), dtype=torch.int64)
    dropped = dev.to_device(np.array([dropped0]), dtype=torch.int64)
    idx_h = np.sort(rs.choice(B, 30, replace=False)).astype(np.int32)[::-1].copy()
    n_rows = 0 if kind == 'max_rows_zero' else 30
    n_acc = dev.to_device(np.array([n_rows]), dtype=torch.int64)
    idx = None if kind == 'null_idx' else dev.to_device(idx_h, dtype=torch.int32)
    arr_p, arr_i = ctypes.c_void_p * 2, ctypes.c_int64 * 2
    ptrs, lds, wid = arr_p(*[s.data_ptr() for s in srcs]), arr_i(*widths), arr_i(*widths)
    cast = lambda a: ctypes.cast(a, ctypes.c_void_p)   # noqa: E731
    _lib.call('elfi_b200_accept_append_f64', dev.context(), dev.ptr(idx), dev.ptr(n_acc),
              0 if kind == 'max_rows_zero' else B, 2, cast(ptrs), cast(lds), cast(wid),
              dev.ptr(dst), ld_dst, capacity, dev.ptr(count),
              None if kind == 'null_dropped' else dev.ptr(dropped), dev.stream_ptr())
    want = np.full((capacity, ld_dst), -7.5)
    rows = min(n_rows, capacity - count0)
    src_rows = np.arange(rows) if kind == 'null_idx' else idx_h[:rows]
    want[count0:count0 + rows, :width] = np.column_stack(srcs_h)[src_rows]
    assert np.array_equal(_host(dst), want)
    assert int(count.item()) == count0 + rows
    lost = n_rows - rows
    assert int(dropped.item()) == dropped0 + (0 if kind == 'null_dropped' else lost)


def _host_model(elfi, batches, obs):
    """The bench's host graph (priors and a 'simulator' handing out host batches, a device
    Distance), restated: each node hands out the next batch of its own list on each call."""
    def feed(values):
        it = iter(values)
        return lambda *args, **kwargs: next(it)

    class Column:
        def __init__(self, values):
            self.rvs = feed(values)

    m = elfi.ElfiModel()
    elfi.Prior(Column([e[0] for _, e in batches]), model=m, name='t1')
    elfi.Prior(Column([e[1] for _, e in batches]), model=m, name='t2')
    elfi.Simulator(feed([S for S, _ in batches]), m['t1'], m['t2'], observed=obs[None, :],
                   name='sim')
    elfi.Summary(lambda x: x, m['sim'], name='S')
    elfi.Distance('euclidean', m['S'], name='d')
    return m


def case_public_rejection():
    """The same host batches through the public elfi_b200.Rejection in threshold mode (its merge
    is merge_topn, another path) and through the bound step: identical d, t1 and t2, ties (a
    repeated batch) included."""
    import elfi_b200 as elfi
    D, B, n = 24, 4000, 700
    rs = np.random.RandomState(700)
    obs = _obs(rs, D)
    layouts = [(1, 'contig'), (1, 'contig')]
    batches = _batches(rs, 4, B, D, layouts, dup={3: 1})
    thr = float(np.quantile(oracle_distances(batches[0][0], obs), 0.1))
    rej = elfi.Rejection(_host_model(elfi, batches, obs)['d'], batch_size=B, seed=1,
                         distributed=False)
    rej.set_objective(n, threshold=thr)
    for _ in batches:
        rej.iterate()
    res = rej.extract_result()
    step = Step(B, D, D, obs, 4 * B, thr, layouts=layouts, thr_mode='host')
    exp = Expected(4 * B, 3)
    run_batches(step, exp, batches, [thr] * 4, obs)
    assert exp.count > n
    top = _host(step.buf.best(n)[0])
    assert np.array_equal(res.discrepancies, top[:, 0])
    assert np.array_equal(res.samples['t1'], top[:, 1])
    assert np.array_equal(res.samples['t2'], top[:, 2])


def case_bench_shape(thr_mode):
    """The bench's step at its scale, its seeded inputs restated: S = RandomState(0).randn(1e6,
    128), obs from RandomState(1), t1 and t2 from RandomState(2), the threshold the 0.01-quantile
    of the distances, four steps over the same batch."""
    B, D, n, steps = 1_000_000, 128, 10_000, 4
    S = np.random.RandomState(0).standard_normal((B, D))
    obs = np.random.RandomState(1).standard_normal((1, D)).ravel()
    rp = np.random.RandomState(2)
    t1, t2 = rp.uniform(-2, 2, B), rp.uniform(-1, 1, B)
    d = oracle_distances(S, obs)
    thr = float(np.quantile(d, 0.01))
    step = Step(B, D, D, obs, B, thr, layouts=[(1, 'contig'), (1, 'contig')], thr_mode=thr_mode)
    exp = Expected(B, 3)
    for _ in range(steps):
        got_d, idx, n_acc = step.batch(S, [t1, t2], thr if thr_mode == 'device' else None)
        want_idx = exp.add(d, [t1, t2], thr)
        assert np.array_equal(got_d, d) and np.array_equal(idx, want_idx)
    assert exp.count == steps * n_acc and exp.dropped == 0
    check_buffer(step, exp)
    top, count, dropped = step.buf.best(n)
    assert (count, dropped) == (steps * n_acc, 0)
    assert np.array_equal(_host(top), exp.merged(thr, n))


def run_largest(stream_ctx=contextlib.nullcontext):
    """case_path_shape at its largest shape inside `stream_ctx`: (d_out, acc_idx, n_acc, rows,
    counters, best) of the last batch as host arrays."""
    with stream_ctx():
        step, exp = case_path_shape(*LARGEST)
        top, count, dropped = step.buf.best(exp.count)
        return [_host(step.d_out), _host(step.acc_idx)[:int(step.n_acc.item())],
                _host(step.buf.rows), _host(step.buf._counters), _host(top)]


def case_refusals():
    """Refused calls raise ElfiB200Error or ValueError and leave the context usable: the next
    valid call gives the same bits.  n_extra = 8, thresholds both on the host and on the device
    or neither, ld_dst below the total width, extras whose widths do not match the buffer,
    thresholds of the wrong count, a source whose columns are not adjacent."""
    import pytest
    from elfi_b200 import _lib, ops
    from elfi_b200 import device as dev
    D, B = 24, 700
    rs = np.random.RandomState(800)
    obs = _obs(rs, D)
    layouts = [(1, 'contig')]
    batches = _batches(rs, 1, B, D, layouts)
    thr = float(np.quantile(oracle_distances(batches[0][0], obs), 0.3))
    step = Step(B, D, D, obs, 2 * B, thr, layouts=layouts)

    def valid():
        step.buf.reset()
        step.buf.rows.fill_(np.nan)
        d, idx, n = step.batch(batches[0][0], batches[0][1], thr)
        return [d, idx, n, _host(step.buf.rows), _host(step.buf._counters)]

    first = valid()
    exp = Expected(2 * B, 2)
    exp.add(oracle_distances(batches[0][0], obs), batches[0][1], thr)
    check_buffer(step, exp)
    errors = (_lib.ElfiB200Error, ValueError)
    Sd, obs_d = step.S, dev.to_device(obs)
    one = dev.to_device(np.zeros(B))

    def same_after(refused):
        with pytest.raises(errors):
            refused()
        again = valid()
        for a, b in zip(first, again):
            assert np.array_equal(a, b, equal_nan=True)

    nine = ops.CandidateBuffer(B, [1] * 9)
    same_after(nine.bind_batch(Sd, obs_d, [thr], step.d_out, step.acc_idx, step.n_acc,
                               [one] * 8))
    arr_p, arr_i = ctypes.c_void_p * 1, ctypes.c_int64 * 1
    ptrs, lds, wid = arr_p(step.extras[0].view.data_ptr()), arr_i(1), arr_i(1)
    cast = lambda a: ctypes.cast(a, ctypes.c_void_p)   # noqa: E731
    thr_h = np.array([thr])

    def rejection_batch(thr_host, thr_dev, ld_dst=2):
        _lib.call('elfi_b200_rejection_batch_f64', dev.context(), dev.ptr(Sd), D, B, D,
                  dev.ptr(obs_d), None, 1, thr_host, thr_dev, dev.ptr(step.d_out),
                  dev.ptr(step.acc_idx), dev.ptr(step.n_acc), 1, cast(ptrs), cast(lds), cast(wid),
                  dev.ptr(step.buf.rows), ld_dst, step.buf.capacity, dev.ptr(step.buf.count),
                  dev.ptr(step.buf.dropped), dev.stream_ptr())
    same_after(lambda: rejection_batch(dev.ptr(thr_h), dev.ptr(step.thr_dev)))
    same_after(lambda: rejection_batch(None, None))
    same_after(lambda: rejection_batch(dev.ptr(thr_h), None, ld_dst=1))
    same_after(lambda: step.buf.bind_batch(Sd, obs_d, [thr], step.d_out, step.acc_idx, step.n_acc,
                                           [dev.empty((B, 2))]))
    same_after(lambda: step.buf.bind_batch(Sd, obs_d, [thr, thr], step.d_out, step.acc_idx,
                                           step.n_acc, [one]))
    same_after(lambda: step.buf.bind_batch(Sd, obs_d, dev.to_device(np.array([thr, thr])),
                                           step.d_out, step.acc_idx, step.n_acc, [one]))
    wide = ops.CandidateBuffer(B, [1, 2])
    same_after(lambda: wide.bind_batch(Sd, obs_d, [thr], step.d_out, step.acc_idx, step.n_acc,
                                       [dev.empty((B, 4))[:, ::2]]))
    same_after(lambda: wide.append([step.d_out, dev.empty((B, 4))[:, ::2]], step.acc_idx,
                                   step.n_acc, B))
