"""The row-stream kernel family of distance.cu and summaries.cu, path by path: a restatement of the
host dispatch, a case table generated from it, and the case bodies shared by
test_rowstream_paths_gpu.py (the device, with the launched kernel observed) and
test_rowstream_paths_cpu_double.py (the CPU test double, which shows that the checkers are sound).

Every result is compared with NumPy / SciPy (the oracle) bit for bit through .view(np.int64), so
signed zeros count; NaN only has to be NaN where the reference is NaN (NaN payloads are not part
of either contract).  General-p Minkowski is held to rtol = 1e-14 (pow accuracy) and the column
moments to the bound derived below.

Dispatch, restated from the C++ (sm = ctx->sm_count, optin = ctx->smem_optin; Dp = D rounded up
to 16; a base is aligned when it is 16-byte aligned):
  tma_compatible(base, ld)  base aligned and ld * 8 % 16 == 0 (ld even)
  rs_aux_offset(ns, w)      (w ns 4096 + w ns 8 + 15) & ~15
  rs_pick_stages(aux, w)    the largest ns in 6 .. 2 with rs_aux_offset(ns, w) + aux + 1024 <= optin
  rs_streams(aux)           D >= 16, tma_compatible and rs_pick_stages(aux, 8) >= 2
Distances (launch_dist), aux = Dp 8 (1 + K with W, else 1):
  rs_streams: W == NULL -> EuclidConsumer; K == 1 -> WeightedConsumer; else NestedConsumer<KMAX>,
  KMAX the first of 2, 3, 4, 5, 6, 8, 16, 32 >= K.  Otherwise dist_direct_kernel.
Distances + column moments (elfi_b200_dist_euclid_mom_f64):
  fused = W != NULL and rs_streams(NestedMomentsConsumer::aux_bytes(Dp, K, 8)),
  aux_bytes(Dp, K, w) = Dp 8 (K + 2 + 2 w).  Fused: NestedMomentsConsumer<KMAX>, KMAX the first of
  2, 4, 6, 8, 16, 32 >= K, at 12 warps when KMAX <= 8 and rs_pick_stages(aux_bytes(Dp, K, 12), 12)
  >= 3 (fused_moments_warps), else at 8; then colmoments_flush_kernel.  Not fused: launch_dist
  as above, then colmoments_partial_kernel / colmoments_final_kernel.
Metrics (launch_metric_t), aux = Dp 8 AUX_ROWS (1; 2 for seuclidean, id 5): rs_streams ->
  MetricConsumer<id>, else metric_direct_kernel<id>.
Segmented distances (launch_seg_t), aux = Dp 8 R: rs_streams -> SegConsumer<id>, else
  seg_direct_kernel<id>.
Autocovariance: rowstream_ok = 16 <= n <= 7688 (PairwiseStream<6>::max_terms()), tma_compatible.
  Lags are taken left to right: (1, 2) as a pair, then 1, 2, 3, 4 alone, each
  AutocovBoxConsumer<LeafSum> when n - LA <= 128 (LEAF_MAX_TERMS), else <TreeSum<6>>; any other
  lag, or not rowstream_ok, goes to summary_direct_kernel.
Mean / variance:
  rowgroup_ok = ld == n, n <= 64, n % 4 == 2, aligned base, rg_smem_bytes(6, 2, n) + 1024 <= optin
    -> meanvar_rowgroup_kernel<NBOX, 8> when rg_smem_bytes(8, 2, n) + 1024 <= optin, else <NBOX, 6>;
    rg_smem_bytes(w, ns, n) = w ns 256 n + 256 + 8 w ns; ns = the largest of 4 .. that fits.
  else rowstream_ok -> MeanVarRegsConsumer<NBOX> (n <= 64), MeanVarBoxConsumer<LeafSum>
    (n <= 128), MeanVarBoxConsumer<TreeSum<6>> (n <= 7688); else summary_direct_kernel.
  NBOX = ceil(n / 16).

Layouts (the leading dimension and the base offset of the input, in doubles): contiguous; ld even
and > D (TMA with a row gap); ld odd; base + 1 (never TMA); base + 2 with ld even (TMA with a
non-zero base); and B = 1, for which the wrappers pass ld = D.  Gaps are filled with a NaN
sentinel, so a kernel that reads outside its row produces NaN.

Row counts: 1 (the B = 1 layout), 33 and 32 k + 7 (a partial last tile), and for every
row-stream path one count at which every warp of the persistent grid consumes more than 2 ns
boxes: it reuses every ring slot at least twice and its mbarrier parity flips (wrap_rows).

Column moments.  Both the fused kernel and colmoments_f64 shift by the first row, d_i = x_i - x_0,
and return mean = x_0 + s1 / n and M2 = s2 - s1^2 / n from s1 = sum d_i, s2 = sum d_i^2 (fma).
With summation depth h (the longest chain of additions any term goes through) and
gamma_k = k u / (1 - k u), u = 2^-53:
  |s1^ - sum d_i| <= gamma_{h+1} sum |d_i|,  |s2^ - sum d_i^2| <= gamma_{h+2} sum d_i^2,
  (sum d_i)^2 / n <= sum d_i^2 (Cauchy-Schwarz), so
  |M2^ - M2| <= 4 gamma_{h+3} sum d_i^2,   |mean^ - mean| <= u |mean| + gamma_{h+2} sum |d_i| / n.
sum d_i^2 = M2 + n (x_0 - mean)^2 and, x_0 being one of the data, (x_0 - mean)^2 <= M2, so
sum d_i^2 <= (n + 1) M2: the shift bounds the cancellation to a factor n + 1 whatever the offset
of the data.  A constant column has every d_i = 0 and M2 = 0.0 exactly.  Depths:
  fused      8 rows per lane + 2 shuffle levels + the tiles a warp owns + ceil(nwarps / 32) + 31
  colmoments ceil(rows_per_block / 8) + 7 + slabs
The reference is a two-pass centred sum in np.longdouble, itself checked against
fractions.Fraction on a small batch.
"""
import ctypes
import fractions
import re
import types
import zlib

import numpy as np
import torch

import elfi_oracle as o
from elfi_b200 import _lib
from elfi_b200 import device as dev

# ---------------------------------------------------------------------------- restatement
RS_WARPS, RS_BOX_ROWS, RS_BOX_COLS, RS_BOX_BYTES, RS_MAX_STAGES = 8, 32, 16, 4096, 6
LEAF_MAX_TERMS = 128
PW_MAX_TERMS = (120 << 6) + 8           # PairwiseStream<6>::max_terms() = 7688
RG_WARPS, RG_SLACK = 8, 256
NESTED_KMAX = (2, 3, 4, 5, 6, 8, 16, 32)
MOM_KMAX = (2, 4, 6, 8, 16, 32)
METRIC_IDS = (1, 2, 3, 4, 5)            # sqeuclidean, cityblock, chebyshev, minkowski, seuclidean
SEG_IDS = (0, 1, 2, 3, 4)
METRIC_NAMES = {0: 'euclidean', 1: 'sqeuclidean', 2: 'cityblock', 3: 'chebyshev', 4: 'minkowski',
                5: 'seuclidean'}
MINKOWSKI_P = 3.5
CONFIGS = {'H100 SXM': (132, 232448), 'H100 PCIe': (114, 232448)}
NOMINAL = CONFIGS['H100 SXM']
CONFIG = list(NOMINAL)    # (sm_count, smem_optin) the bodies assume; the device tests set the live one


def padded(D):
    return -(-D // RS_BOX_COLS) * RS_BOX_COLS


def rs_aux_offset(ns, warps=RS_WARPS):
    return (warps * ns * RS_BOX_BYTES + warps * ns * 8 + 15) & ~15


def rs_pick_stages(optin, aux, warps=RS_WARPS):
    for ns in range(RS_MAX_STAGES, 1, -1):
        if rs_aux_offset(ns, warps) + aux + 1024 <= optin:
            return ns
    return 0


def tma_compatible(aligned, ld):
    return aligned and (ld * 8) % 16 == 0


def rs_streams(optin, aligned, ld, D, aux):
    return D >= RS_BOX_COLS and tma_compatible(aligned, ld) and rs_pick_stages(optin, aux) >= 2


def mom_aux_bytes(Dp, K, warps=RS_WARPS):
    return Dp * 8 * (1 + K + 1 + 2 * warps)


def fused_moments_warps(optin, KMAX, Dp, K):
    if KMAX > 8:
        return RS_WARPS
    return 12 if rs_pick_stages(optin, mom_aux_bytes(Dp, K, 12), 12) >= 3 else RS_WARPS


def rg_smem_bytes(warps, ns, n):
    return warps * ns * 32 * n * 8 + RG_SLACK + warps * ns * 8


def rowgroup_ok(optin, aligned, ld, n):
    return ld == n and n <= 64 and n % 4 == 2 and aligned and rg_smem_bytes(6, 2, n) + 1024 <= optin


def rowgroup_warps(optin, n):
    return RG_WARPS if rg_smem_bytes(RG_WARPS, 2, n) + 1024 <= optin else 6


def rowgroup_stages(optin, warps, n):
    ns = 4
    while rg_smem_bytes(warps, ns, n) + 1024 > optin:
        ns -= 1
    return ns


def summary_rowstream_ok(optin, aligned, ld, n):
    return RS_BOX_COLS <= n <= PW_MAX_TERMS and tma_compatible(aligned, ld) and \
        rs_pick_stages(optin, 0) >= 2


def first_at_least(values, K):
    return next(v for v in values if v >= K)


# ---------------------------------------------------------------------------- registry
class Path(types.SimpleNamespace):
    """name; kernel: the substring of the launched kernel's demangled name (whitespace and '(int)'
    removed); consumer: the key the source scan finds."""


def _rs(consumer, warps=RS_WARPS):
    return 'rowstream_kernel<elfi::{},{}>'.format(consumer, warps)


def _registry():
    P = []

    def add(name, kernel, consumer):
        P.append(Path(name=name, kernel=kernel, consumer=consumer))
    add('dist:Euclid', _rs('EuclidConsumer'), 'EuclidConsumer')
    add('dist:Weighted', _rs('WeightedConsumer'), 'WeightedConsumer')
    for k in NESTED_KMAX:
        add('dist:Nested<{}>'.format(k), _rs('NestedConsumer<{}>'.format(k)),
            'NestedConsumer<{}>'.format(k))
    add('dist:direct', 'elfi::dist_direct_kernel(', 'dist_direct_kernel')
    for k in MOM_KMAX:
        for w in ((12, 8) if k <= 8 else (8,)):
            add('mom:NestedMoments<{}>/{}w'.format(k, w), _rs('NestedMomentsConsumer<{}>'.format(k), w),
                'NestedMomentsConsumer<{}>'.format(k))
    add('mom:colmoments', 'elfi::colmoments_partial_kernel(', 'colmoments')
    for m in METRIC_IDS:
        add('metric:Metric<{}>'.format(m), _rs('MetricConsumer<{}>'.format(m)),
            'MetricConsumer<{}>'.format(m))
        add('metric:direct<{}>'.format(m), 'elfi::metric_direct_kernel<{}>('.format(m),
            'metric_direct_kernel<{}>'.format(m))
    for m in SEG_IDS:
        add('seg:Seg<{}>'.format(m), _rs('SegConsumer<{}>'.format(m)), 'SegConsumer<{}>'.format(m))
        add('seg:direct<{}>'.format(m), 'elfi::seg_direct_kernel<{}>('.format(m),
            'seg_direct_kernel<{}>'.format(m))
    for la, lb in ((1, 2), (1, -1), (2, -1), (3, -1), (4, -1)):
        for sname, sk in (('Leaf', 'elfi::LeafSum'), ('Tree', 'elfi::TreeSum<6>')):
            add('autocov:{}<{},{}>'.format(sname, la, lb),
                _rs('AutocovBoxConsumer<{},{},{}>'.format(sk, la, lb)),
                'AutocovBoxConsumer<{},{},{}>'.format(sname, la, lb))
    add('summary:direct', 'elfi::summary_direct_kernel(', 'summary_direct_kernel')
    for nb in (1, 2, 3, 4):
        for w in (8, 6):
            add('meanvar:rowgroup<{},{}>'.format(nb, w),
                'elfi::meanvar_rowgroup_kernel<{},{}>('.format(nb, w), 'rowgroup<{},{}>'.format(nb, w))
        add('meanvar:Regs<{}>'.format(nb), _rs('MeanVarRegsConsumer<{}>'.format(nb)),
            'MeanVarRegsConsumer<{}>'.format(nb))
    add('meanvar:BoxLeaf', _rs('MeanVarBoxConsumer<elfi::LeafSum>'), 'MeanVarBoxConsumer<Leaf>')
    add('meanvar:BoxTree', _rs('MeanVarBoxConsumer<elfi::TreeSum<6>>'), 'MeanVarBoxConsumer<Tree>')
    return {p.name: p for p in P}


REGISTRY = _registry()


def reachable(optin):
    """Registry paths some input selects at this shared-memory opt-in.  The row-group kernel's
    warp count depends on n and optin alone: at 227 KiB only NBOX = 4 (n = 58, 62) needs 6 warps."""
    rg = {'meanvar:rowgroup<{},{}>'.format(-(-n // 16), rowgroup_warps(optin, n))
          for n in range(2, 65, 4) if rowgroup_ok(optin, True, n, n)}
    return sorted(n for n in REGISTRY if not n.startswith('meanvar:rowgroup') or n in rg)


def normalize_kernel_name(name):
    return re.sub(r'\s+', '', name).replace('(int)', '')


def paths_in(kernel_names):
    """Registry paths whose kernel appears among the launched kernel names."""
    names = [normalize_kernel_name(k) for k in kernel_names]
    return {p.name for p in REGISTRY.values() if any(p.kernel in k for k in names)}


# ---------------------------------------------------------------------------- prediction
def predict(case, optin):
    """The set of registry paths a case launches, from the restated dispatch."""
    aligned = case.off % 2 == 0
    ld = case.ld
    f = case.family
    if f == 'dist':
        return {_predict_dist(optin, aligned, ld, case.D, case.K, case.weighted)}
    if f == 'mom':
        D, K = case.D, case.K
        Dp = padded(D)
        if case.weighted and rs_streams(optin, aligned, ld, D, mom_aux_bytes(Dp, K)):
            kmax = first_at_least(MOM_KMAX, K)
            return {'mom:NestedMoments<{}>/{}w'.format(kmax, fused_moments_warps(optin, kmax, Dp, K))}
        return {'mom:colmoments', _predict_dist(optin, aligned, ld, D, K, case.weighted)}
    if f == 'metric':
        aux = padded(case.D) * 8 * (2 if case.metric == 5 else 1)
        kind = 'Metric' if rs_streams(optin, aligned, ld, case.D, aux) else 'direct'
        return {'metric:{}<{}>'.format(kind, case.metric)}
    if f == 'seg':
        aux = padded(case.D) * 8 * case.R
        kind = 'Seg' if rs_streams(optin, aligned, ld, case.D, aux) else 'direct'
        return {'seg:{}<{}>'.format(kind, case.metric)}
    if f == 'autocov':
        return _predict_autocov(optin, aligned, ld, case.D, case.lags)
    if f == 'meanvar':
        return {_predict_meanvar(optin, aligned, ld, case.D)}
    raise ValueError(f)


def _predict_dist(optin, aligned, ld, D, K, weighted):
    aux = padded(D) * 8 * ((1 + K) if weighted else 1)
    if not rs_streams(optin, aligned, ld, D, aux):
        return 'dist:direct'
    if not weighted:
        return 'dist:Euclid'
    if K == 1:
        return 'dist:Weighted'
    return 'dist:Nested<{}>'.format(first_at_least(NESTED_KMAX, K))


def _predict_autocov(optin, aligned, ld, n, lags):
    fast = summary_rowstream_ok(optin, aligned, ld, n)
    out, l = set(), 0
    while l < len(lags):
        la = lags[l]
        lb = lags[l + 1] if l + 1 < len(lags) else -1
        if fast and la in (1, 2, 3, 4):
            pair = la == 1 and lb == 2
            kind = 'Leaf' if n - la <= LEAF_MAX_TERMS else 'Tree'
            out.add('autocov:{}<{},{}>'.format(kind, la, 2 if pair else -1))
            l += 2 if pair else 1
        else:
            out.add('summary:direct')
            l += 1
    return out


def _predict_meanvar(optin, aligned, ld, n):
    if rowgroup_ok(optin, aligned, ld, n):
        return 'meanvar:rowgroup<{},{}>'.format(-(-n // 16), rowgroup_warps(optin, n))
    if summary_rowstream_ok(optin, aligned, ld, n):
        if n <= 64:
            return 'meanvar:Regs<{}>'.format(-(-n // 16))
        return 'meanvar:BoxLeaf' if n <= LEAF_MAX_TERMS else 'meanvar:BoxTree'
    return 'summary:direct'


def primary(case, optin):
    """The first of the case's predicted paths, leaving out the stand-alone column moments."""
    return sorted(p for p in predict(case, optin) if p != 'mom:colmoments')[0]


def ring(case, optin):
    """(warps, stages, boxes per tile) of the persistent ring the case's primary path runs, or
    None for a thread-per-row kernel."""
    path = primary(case, optin)
    D = case.D
    Gc = -(-D // RS_BOX_COLS)
    if 'direct' in path:
        return None
    if path.startswith('meanvar:rowgroup'):
        w = rowgroup_warps(optin, D)
        return w, rowgroup_stages(optin, w, D), 1
    if path.startswith('mom:'):
        kmax = int(re.search(r'<(\d+)>', path).group(1))
        w = fused_moments_warps(optin, kmax, padded(D), case.K)
        return w, rs_pick_stages(optin, mom_aux_bytes(padded(D), case.K, w), w), Gc
    if path.startswith('dist:'):
        aux = padded(D) * 8 * ((1 + case.K) if case.weighted else 1)
    elif path.startswith('metric:'):
        aux = padded(D) * 8 * (2 if case.metric == 5 else 1)
    elif path.startswith('seg:'):
        aux = padded(D) * 8 * case.R
    else:
        aux = 0
    passes = 2 if path.startswith('meanvar:Box') else 1
    return RS_WARPS, rs_pick_stages(optin, aux), Gc * passes


def wrap_rows(case, sm, optin):
    """Rows at which every warp of the persistent grid consumes more than 2 ns boxes (+ 7: a
    partial last tile)."""
    w, ns, G = ring(case, optin)
    tiles_per_warp = -(-(2 * ns + 1) // G)
    return RS_BOX_ROWS * sm * w * tiles_per_warp + 7


# ---------------------------------------------------------------------------- the case table
LAYOUTS = ('contig', 'ld_even', 'ld_odd', 'off1', 'off2', 'b1')
THRESHOLD_LAYOUTS = ('contig', 'ld_even', 'off2', 'b1')


def layout(D, name):
    """(ld, base offset in doubles) of a layout for rows of D."""
    even_gap = D + 2 if D % 2 == 0 else D + 1
    odd_gap = D + 1 if D % 2 == 0 else D + 2
    return {'contig': (D, 0), 'ld_even': (even_gap, 0), 'ld_odd': (odd_gap, 0),
            'off1': (D, 1), 'off2': (D if D % 2 == 0 else D + 1, 2), 'b1': (D, 0)}[name]


def _max_streaming_D(optin, per_col_rows):
    """Largest D whose row-stream aux (Dp 8 per_col_rows bytes) still leaves a 2-slot ring."""
    Dp = 16
    while rs_pick_stages(optin, (Dp + 16) * 8 * per_col_rows) >= 2:
        Dp += 16
    return Dp


def _max_D(pred):
    Dp = 16
    while pred(Dp + 16):
        Dp += 16
    return Dp


def _shapes(optin):
    """(family, params, threshold) candidates: small shapes for every layout, and the shapes on
    both sides of every shared-memory and row-length threshold."""
    S = []
    # distances
    for weighted, K in [(False, 1), (True, 1)] + [(True, k) for k in (2, 3, 4, 5, 6, 7, 8, 9, 16, 17, 32)]:
        for D in (7, 16, 33):
            S.append(('dist', dict(D=D, K=K, weighted=weighted), False))
        Dm = _max_streaming_D(optin, (1 + K) if weighted else 1)
        if K in (1, 16, 32):
            S += [('dist', dict(D=Dm, K=K, weighted=weighted), True),
                  ('dist', dict(D=Dm + 1, K=K, weighted=weighted), True)]
    # distances + moments
    for K in (1, 2, 3, 4, 5, 6, 7, 8, 9, 16, 17, 32):
        for D in (7, 16, 33):
            S.append(('mom', dict(D=D, K=K, weighted=True), False))
        d8 = _max_D(lambda Dp: rs_pick_stages(optin, mom_aux_bytes(Dp, K)) >= 2)
        S += [('mom', dict(D=d8, K=K, weighted=True), True),
              ('mom', dict(D=d8 + 1, K=K, weighted=True), True)]
        if K <= 8:
            d12 = _max_D(lambda Dp: rs_pick_stages(optin, mom_aux_bytes(Dp, K, 12), 12) >= 3)
            S += [('mom', dict(D=d12, K=K, weighted=True), True),
                  ('mom', dict(D=d12 + 1, K=K, weighted=True), True)]
    S.append(('mom', dict(D=16, K=1, weighted=False), False))
    # metrics
    for m in METRIC_IDS:
        for D in (7, 16, 33):
            S.append(('metric', dict(D=D, metric=m), False))
        Dm = _max_streaming_D(optin, 2 if m == 5 else 1)
        S += [('metric', dict(D=Dm, metric=m), True), ('metric', dict(D=Dm + 1, metric=m), True)]
    # segmented distances: a tile of 32 rows straddles segments of 5 rows
    for m in SEG_IDS:
        for D in (7, 16, 33):
            S.append(('seg', dict(D=D, metric=m, R=3), False))
        Rm = _max_streaming_D(optin, 1) // 16
        S += [('seg', dict(D=16, metric=m, R=Rm), True), ('seg', dict(D=16, metric=m, R=Rm + 1), True)]
    # autocovariance
    for lags in ((1, 2), (1,), (2,), (3,), (4,), (5,)):
        for n in (15, 16, 37, 100):
            S.append(('autocov', dict(D=n, lags=lags), False))
        la = lags[0]
        for n in (LEAF_MAX_TERMS + la, LEAF_MAX_TERMS + la + 1, PW_MAX_TERMS, PW_MAX_TERMS + 1):
            S.append(('autocov', dict(D=n, lags=lags), True))
    for lags in ((2, 1), (1, 2, 3, 7)):
        S.append(('autocov', dict(D=100, lags=lags), False))
    # mean / variance: every n = 2 mod 4 of the row-group kernel, the register consumers' ends
    rg6 = min(n for n in range(2, 65, 4) if rowgroup_warps(optin, n) == 6)
    for n in sorted({2, 6, 14, 15, 16, 17, 18, 20, 30, 32, 34, 36, 46, 48, 50, rg6 - 4, rg6, 62, 64, 65}):
        S.append(('meanvar', dict(D=n), False))
    for n in (LEAF_MAX_TERMS, LEAF_MAX_TERMS + 1, PW_MAX_TERMS, PW_MAX_TERMS + 1):
        S.append(('meanvar', dict(D=n), True))
    return S


class Case(types.SimpleNamespace):
    def ident(self):
        extra = ''
        if self.family in ('dist', 'mom'):
            extra = '-K{}{}'.format(self.K, '' if self.weighted else 'u')
        elif self.family in ('metric', 'seg'):
            extra = '-m{}'.format(self.metric) + ('-R{}'.format(self.R) if self.family == 'seg' else '')
        elif self.family == 'autocov':
            extra = '-lags' + '_'.join(str(l) for l in self.lags)
        return '{}{}-D{}-{}-B{}'.format(self.family, extra, self.D, self.layout, self.B)


def table(sm, optin):
    """Every case of the family, generated from the restatement.  Small shapes run in every
    layout (33 or 32 k + 7 rows, alternately; 1 row for 'b1'), threshold shapes in every layout
    that can stream (contiguous, an even row gap -- odd n streams only with one --, an aligned
    non-zero base, B = 1), and every row-stream path once more at its wrap row count, at the
    narrowest input that selects it."""
    out = []
    for fam, prm, threshold in _shapes(optin):
        D = prm['D']
        for i, lay in enumerate(THRESHOLD_LAYOUTS if threshold else LAYOUTS):
            ld, off = layout(D, lay)
            if fam == 'seg':
                rows = prm['R'] * (1 if lay == 'b1' or threshold else 5 + 2 * (i % 2))
            else:
                rows = 1 if lay == 'b1' else (33 if i % 2 == 0 else 32 * 5 + 7)
            out.append(Case(family=fam, layout=lay, ld=ld, off=off, B=rows, wrap=False, **prm))
    seen = set()
    for c in sorted(out, key=lambda c: (c.D, c.B)):     # each path's wrap case at its narrowest rows
        key = primary(c, optin)
        if key in seen or c.layout not in ('contig', 'ld_even') or ring(c, optin) is None:
            continue
        if c.family == 'seg' and c.R > 3:
            continue
        seen.add(key)
        w = Case(**dict(vars(c)))
        w.B = wrap_rows(c, sm, optin)
        if w.family == 'seg':
            w.B -= w.B % w.R
        w.wrap = True
        out.append(w)
    return out


def layout_gaps(cases, optin):
    """(path, layout) pairs a path admits but no case runs: a case of the path whose shape, laid
    out in another layout, still selects the path, shows that the path admits that layout."""
    have, admits = set(), set()
    for c in cases:
        p = primary(c, optin)
        have.add((p, c.layout))
        for lay in LAYOUTS:
            ld, off = layout(c.D, lay)
            moved = Case(**dict(vars(c), layout=lay, ld=ld, off=off))
            if primary(moved, optin) == p:
                admits.add((p, lay))
    return sorted(admits - have)


def representatives(cases, optin):
    """One small case per path: the fewest doubles of input among the cases that launch it."""
    rep = {}
    for c in sorted(cases, key=lambda c: (c.B * c.D, c.ident())):
        for p in predict(c, optin):
            rep.setdefault(p, c)
    return rep


def uncovered(sm, optin):
    covered = set()
    for c in table(sm, optin):
        covered |= predict(c, optin)
    return sorted(set(reachable(optin)) - covered)


# ---------------------------------------------------------------------------- the source scan
def scan_sources(distance_cu, summaries_cu):
    """Consumer / kernel keys that distance.cu and summaries.cu launch: every consumer passed to
    rowstream_launch<...> (template arguments kept when they are literals; the typedef of
    launch_metric_t resolved), every *_direct_kernel<<<, every meanvar_rowgroup_kernel instance,
    and 'colmoments' for a call of the stand-alone column moments."""
    keys = set()
    for text in (distance_cu, summaries_cu):
        if re.search(r'\belfi_b200_colmoments_f64\(', text):
            keys.add('colmoments')
        typedefs = dict((b, a) for a, b in re.findall(r'typedef\s+(\w+)<[^;]*>\s+(\w+);', text))
        for name, args in re.findall(r'rowstream_launch<\s*(\w+)\s*(<[^<>]*(?:<[^<>]*>[^<>]*)*>)?', text):
            name = typedefs.get(name, name)
            a = re.sub(r'\s+', '', args or '')
            literal = a and all(re.fullmatch(r'-?\d+', x) for x in a[1:-1].split(','))
            keys.add(name + a if literal else name)
        for name in re.findall(r'(\w+_direct_kernel)(?:<\w+>)?\s*<<<', text):
            keys.add(name)
        nboxes = re.findall(r'rowgroup_launch<(\d+)>\(', text)
        warps = re.findall(r'rowgroup_launch_w<NBOX,\s*(\w+)>', text)
        consts = dict(re.findall(r'constexpr int (\w+) = (\d+);', text))
        for nb in nboxes:
            for w in warps:
                keys.add('rowgroup<{},{}>'.format(nb, consts.get(w, w)))
    return keys


def names(key, consumer):
    """Does a scanned key name a registry consumer (by instance, or by template name)?"""
    return key == consumer or ('<' not in key and consumer.split('<')[0] == key)


def registry_has(key):
    return any(names(key, p.consumer) for p in REGISTRY.values())


def launched(keys, consumer):
    return any(names(k, consumer) for k in keys)


# ---------------------------------------------------------------------------- data
SENTINEL = np.array([0x7FF4DEADBEEF0001], dtype=np.int64).view(np.float64)[0]


def data(B, D, seed, specials=True):
    """(B, D) rows with columns scaled by 10^U(-3, 3), and, from row 1 on, a NaN, +-inf, and
    rows of +0.0, -0.0 and mixed signed zeros."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, D, generator=g, dtype=torch.float64).numpy()
    scale = 10.0 ** np.random.RandomState(seed).uniform(-3, 3, D)
    x *= scale
    if specials and B >= 8:
        x[1, D // 2] = np.nan
        x[2, min(1, D - 1)] = np.inf
        x[3, D - 1] = -np.inf
        x[4] = 0.0
        x[5] = -0.0
        x[6, ::2] = -0.0
        x[6, 1::2] = 0.0
    return x, scale


def place(x, ld, off):
    """Device buffer holding x with leading dimension ld at base offset off (doubles), NaN
    sentinel in every gap; returns (buffer, pointer)."""
    B, D = x.shape
    flat = np.full(off + max(B - 1, 0) * ld + D + 2, SENTINEL)
    rows = np.lib.stride_tricks.as_strided(flat[off:], (B, D), (ld * 8, 8))
    rows[...] = x
    buf = dev.to_device(flat)
    return buf, ctypes.c_void_p(buf.data_ptr() + 8 * off)


def sentinel_buffer(shape):
    return dev.full(shape, SENTINEL)


def host(t):
    return t.cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


def same_bits(got, ref, what):
    got, ref = np.asarray(got, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    assert got.shape == ref.shape, what
    assert not np.any(got.view(np.int64) == SENTINEL.view(np.int64)), what + ': cell not written'
    nan_g, nan_r = np.isnan(got), np.isnan(ref)
    bad = (nan_g != nan_r) | (~nan_r & (got.view(np.int64) != ref.view(np.int64)))
    if bad.any():
        i = np.argwhere(bad)[:5]
        raise AssertionError('{}: {} of {} differ, first at {}: got {} want {}'.format(
            what, int(bad.sum()), bad.size, i.tolist(), got[tuple(i[0])], ref[tuple(i[0])]))


def close(got, ref, rtol, what):
    got, ref = np.asarray(got), np.asarray(ref)
    same_special = np.array_equal(np.isnan(got), np.isnan(ref)) and \
        np.array_equal(np.where(np.isinf(ref), ref, 0), np.where(np.isinf(got), got, 0))
    fin = np.isfinite(ref)
    ok = same_special and np.all(np.abs(got[fin] - ref[fin]) <= rtol * np.abs(ref[fin]))
    assert ok, '{}: beyond rtol {}'.format(what, rtol)


def untouched(buf, mask, what):
    b = host(buf)
    assert np.all(b[mask].view(np.int64) == SENTINEL.view(np.int64)), what + ': wrote outside'
    assert not np.any(b[~mask].view(np.int64) == SENTINEL.view(np.int64)), what + ': cell not written'


# ---------------------------------------------------------------------------- case bodies
def run(case):
    """Run one case through the C ABI and check every output against the host reference."""
    return {'dist': _run_dist, 'mom': _run_dist, 'metric': _run_metric, 'seg': _run_seg,
            'autocov': _run_autocov, 'meanvar': _run_meanvar}[case.family](case)


def _seed(case, salt):
    return zlib.crc32('{}/{}'.format(case.ident(), salt).encode())


def _thr(d, K):
    fin = np.where(np.isfinite(d), d, np.nan).reshape(len(d), K)
    q = np.nanquantile(fin, 0.4, axis=0) if np.isfinite(fin).any() else np.zeros(K)
    return np.ascontiguousarray(np.where(np.isfinite(q), q, 0.0))


def _accepted(d, thr):
    return np.nonzero(np.all(d.reshape(len(d), -1) <= thr, axis=1))[0]


def _check_accept(d, thr, idx, n_acc, what):
    want = _accepted(d, thr)
    n = int(host(n_acc)[0])
    assert n == len(want), '{}: {} accepted, want {}'.format(what, n, len(want))
    assert np.array_equal(host(idx)[:n], want), what + ': accepted set'


def _run_dist(c):
    B, D, K = c.B, c.D, c.K
    seed = _seed(c, 1)
    x, scale = data(B, D, seed)
    obs = np.random.RandomState(seed + 1).randn(D) * scale
    W = (10.0 ** np.random.RandomState(seed + 2).uniform(-1, 1, (K, D))) / scale ** 2 \
        if c.weighted else None
    buf, S = place(x, c.ld, c.off)
    ref = np.column_stack([o.cdist_euclid(x, obs, w=None if W is None else W[k]) for k in range(K)])
    thr = _thr(ref, K)
    obs_d = dev.to_device(obs)
    W_d = None if W is None else dev.to_device(W)
    d_out = sentinel_buffer((B, K))
    idx = dev.full((B,), -1, dtype=torch.int32)
    n_acc = dev.zeros((1,), dtype=torch.int64)
    if c.family == 'mom':
        mom = sentinel_buffer((2, D))
        _lib.call('elfi_b200_dist_euclid_mom_f64', dev.context(), S, c.ld, B, D, dev.ptr(obs_d),
                  dev.ptr(W_d), K, thr.ctypes.data_as(ctypes.c_void_p), None, dev.ptr(d_out),
                  dev.ptr(idx), dev.ptr(n_acc), dev.ptr(mom), dev.stream_ptr())
    else:
        _lib.call('elfi_b200_dist_euclid_thr_f64', dev.context(), S, c.ld, B, D, dev.ptr(obs_d),
                  dev.ptr(W_d), K, thr.ctypes.data_as(ctypes.c_void_p), dev.ptr(d_out),
                  dev.ptr(idx), dev.ptr(n_acc), dev.stream_ptr())
    dev.synchronize()
    d = host(d_out)
    same_bits(d, ref, c.ident() + ' d')
    _check_accept(d, thr, idx, n_acc, c.ident())
    if c.family == 'mom':
        m = host(mom)
        check_moments(x, m[0], m[1], moments_depth(c, B), c.ident())


def _run_metric(c):
    B, D, m = c.B, c.D, c.metric
    seed = _seed(c, 2)
    x, scale = data(B, D, seed)
    obs = np.random.RandomState(seed + 1).randn(D) * scale
    buf, S = place(x, c.ld, c.off)
    d_out = sentinel_buffer((B,))
    idx = dev.full((B,), -1, dtype=torch.int32)
    n_acc = dev.zeros((1,), dtype=torch.int64)
    obs_d = dev.to_device(obs)
    if m == 5:
        V = 10.0 ** np.random.RandomState(seed + 3).uniform(-1, 1, D) * scale ** 2
        ref = o.cdist_seuclidean(x, obs, V)
        thr = _thr(ref, 1)
        V_d = dev.to_device(V)
        _lib.call('elfi_b200_dist_seuclidean_thr_f64', dev.context(), S, c.ld, B, D, dev.ptr(obs_d),
                  dev.ptr(V_d), thr.ctypes.data_as(ctypes.c_void_p), dev.ptr(d_out), dev.ptr(idx),
                  dev.ptr(n_acc), dev.stream_ptr())
    else:
        ref = o.cdist_metric(x, obs, METRIC_NAMES[m], MINKOWSKI_P)
        thr = _thr(ref, 1)
        _lib.call('elfi_b200_dist_metric_thr_f64', dev.context(), m, MINKOWSKI_P, S, c.ld, B, D,
                  dev.ptr(obs_d), thr.ctypes.data_as(ctypes.c_void_p), dev.ptr(d_out), dev.ptr(idx),
                  dev.ptr(n_acc), dev.stream_ptr())
    dev.synchronize()
    d = host(d_out)
    if m == 4:
        close(d, ref, 1e-14, c.ident())
    else:
        same_bits(d, ref, c.ident())
    _check_accept(d, thr, idx, n_acc, c.ident())


def seg_reference(x, O, R, metric):
    rows = len(x) // R
    out = []
    for r in range(R):
        seg = x[r * rows:(r + 1) * rows]
        out.append(o.cdist_euclid(seg, O[r]) if metric == 0 else
                   o.cdist_metric(seg, O[r], METRIC_NAMES[metric], MINKOWSKI_P))
    return np.concatenate(out)


def _run_seg(c):
    B, D, R, m = c.B, c.D, c.R, c.metric
    seed = _seed(c, 3)
    x, scale = data(B, D, seed)
    O = np.random.RandomState(seed + 1).randn(R, D) * scale
    ld_obs = D + 3
    obuf, Op = place(O, ld_obs, 0)
    buf, S = place(x, c.ld, c.off)
    d_out = sentinel_buffer((B,))
    _lib.call('elfi_b200_dist_seg_f64', dev.context(), m, MINKOWSKI_P, S, c.ld, R, B // R, D, Op,
              ld_obs, dev.ptr(d_out), dev.stream_ptr())
    dev.synchronize()
    ref = seg_reference(x, O, R, m)
    if m == 4:
        close(host(d_out), ref, 1e-14, c.ident())
    else:
        same_bits(host(d_out), ref, c.ident())


def autocov_reference(x, lag):
    return np.mean(x[:, lag:] * x[:, :-lag], axis=1)


def _run_autocov(c):
    B, n, lags = c.B, c.D, c.lags
    x, _ = data(B, n, _seed(c, 4))
    buf, X = place(x, c.ld, c.off)
    nl = len(lags)
    ld_out = nl + 2                       # two columns the call must leave alone
    out = sentinel_buffer((B, ld_out))
    lags_h = np.ascontiguousarray(lags, dtype=np.int32)
    _lib.call('elfi_b200_summary_autocov_f64', dev.context(), X, c.ld, B, n,
              lags_h.ctypes.data_as(ctypes.c_void_p), nl, dev.ptr(out), ld_out, dev.stream_ptr())
    dev.synchronize()
    got = host(out)
    with np.errstate(all='ignore'):
        ref = np.column_stack([autocov_reference(x, l) for l in lags])
    same_bits(got[:, :nl], ref, c.ident())
    mask = np.zeros(got.shape, dtype=bool)
    mask[:, nl:] = True
    untouched(out, mask, c.ident())


def meanvar_reference(x):
    with np.errstate(all='ignore'):
        return np.mean(x, axis=1), np.var(x, axis=1)


def _run_meanvar(c, col_mean=0, col_var=1, ld_out=3):
    B, n = c.B, c.D
    x, _ = data(B, n, _seed(c, 5))
    buf, X = place(x, c.ld, c.off)
    out = sentinel_buffer((B, ld_out))
    _lib.call('elfi_b200_summary_meanvar_f64', dev.context(), X, c.ld, B, n, dev.ptr(out), ld_out,
              col_mean, col_var, dev.stream_ptr())
    dev.synchronize()
    got = host(out)
    mean, var = meanvar_reference(x)
    mask = np.ones(got.shape, dtype=bool)
    if col_mean >= 0:
        same_bits(got[:, col_mean], mean, c.ident() + ' mean')
        mask[:, col_mean] = False
    if col_var >= 0:
        same_bits(got[:, col_var], var, c.ident() + ' var')
        mask[:, col_var] = False
    untouched(out, mask, c.ident())


def meanvar_columns(case, col_mean, col_var, ld_out):
    _run_meanvar(case, col_mean, col_var, ld_out)


# ---------------------------------------------------------------------------- column moments
U = 2.0 ** -53


def gamma(k):
    return k * U / (1 - k * U)


def moments_depth(case, B, sm=None, optin=None):
    """Summation depth h of the column moments the case's path computes (module docstring)."""
    sm = CONFIG[0] if sm is None else sm
    optin = CONFIG[1] if optin is None else optin
    paths = predict(case, optin)
    fused = [p for p in paths if p.startswith('mom:NestedMoments')]
    if fused:
        w = int(re.search(r'/(\d+)w', fused[0]).group(1))
        ntiles = -(-B // RS_BOX_ROWS)
        ctas = min(-(-ntiles // w), sm)
        nwarps = ctas * w
        return 8 + 2 + -(-ntiles // nwarps) + -(-nwarps // 32) + 31
    return colmoments_depth(case.D, B, sm)


def colmoments_depth(D, B, sm):
    """Summation depth of colmoments_partial_kernel + colmoments_final_kernel: a chain of
    ceil(R / 8) rows, 7 adds across the chains of a block, then the blocks in order."""
    colgroups = -(-D // 32)
    slabs = -(-(sm * 8) // colgroups)
    rpb = max(-(-B // slabs), 64)
    slabs = -(-B // rpb)
    return -(-rpb // 8) + 7 + slabs


def exact_moments(x):
    """Two-pass centred (mean, M2, sum |x - x0|, sum (x - x0)^2) per column in np.longdouble."""
    xl = np.asarray(x, dtype=np.longdouble)
    d = xl - xl[0]
    n = xl.shape[0]
    mean_d = d.sum(axis=0) / n
    return xl[0] + mean_d, ((d - mean_d) ** 2).sum(axis=0), np.abs(d).sum(axis=0), (d * d).sum(axis=0)


def fraction_moments(x):
    n = x.shape[0]
    means, m2 = [], []
    for j in range(x.shape[1]):
        col = [fractions.Fraction(float(v)) for v in x[:, j]]
        mu = sum(col) / n
        means.append(mu)
        m2.append(sum((v - mu) ** 2 for v in col))
    return means, m2


def check_moments(x, mean, m2, h, what):
    """The fused / stand-alone moments against the bound of the module docstring.  Columns with a
    non-finite entry only have to be non-finite."""
    fin = np.all(np.isfinite(x), axis=0)
    assert not np.any(np.isfinite(m2[~fin])), what + ': a column with NaN / inf has a finite M2'
    if not fin.any():
        return
    xm = x[:, fin]
    ref_mean, ref_m2, sabs, s2 = exact_moments(xm)
    n = xm.shape[0]
    tol_mean = U * np.abs(ref_mean) + gamma(h + 2) * sabs / n
    tol_m2 = 4 * gamma(h + 3) * s2
    err_mean = np.abs(np.asarray(mean[fin], dtype=np.longdouble) - ref_mean)
    err_m2 = np.abs(np.asarray(m2[fin], dtype=np.longdouble) - ref_m2)
    assert np.all(err_mean <= tol_mean), '{}: mean error {} > bound {}'.format(
        what, float(np.max(err_mean - tol_mean)), float(np.max(tol_mean)))
    assert np.all(err_m2 <= tol_m2), '{}: M2 error ratio {}'.format(
        what, float(np.max(err_m2 / np.where(tol_m2 > 0, tol_m2, 1))))
    assert np.all(s2 <= (n + 1) * ref_m2 * (1 + 1e-12) + 1e-300), what + ': sum d^2 > (n + 1) M2'
    zero = ref_m2 == 0
    assert np.all(m2[fin][zero] == 0.0), what + ': constant column with M2 != 0'


ACCURACY_KINDS = ('outlier_first_row', 'offset_1e8', 'constant', 'single_row', 'partial_tile')


def accuracy_data(kind, D=48):
    rs = np.random.RandomState(len(kind))
    if kind == 'outlier_first_row':
        x = rs.randn(100_003, D)
        x[0] = 1e4
    elif kind == 'offset_1e8':
        x = 1e8 + rs.randn(50_001, D)
    elif kind == 'constant':
        x = rs.randn(4_099, D)
        x[:, ::3] = 7.25
    elif kind == 'single_row':
        x = rs.randn(1, D)
    else:
        x = rs.randn(32 * 77 + 19, D) * 10.0 ** rs.uniform(-3, 3, D)
    return x


MOMENT_ROUTES = {'fused12': 2, 'fused8': 9, 'colmoments': 2}   # route -> K (9: KMAX 16, 8 warps)


def moments_accuracy(kind, route, D=48):
    """The column moments of accuracy_data(kind) through the fused kernel at 12 or 8 warps, or the
    stand-alone colmoments_f64, against check_moments' bound; returns the case (for its path)."""
    K = MOMENT_ROUTES[route]
    x = accuracy_data(kind, D)
    B = x.shape[0]
    buf, S = place(x, D, 0)
    mom = sentinel_buffer((2, D))
    c = Case(family='mom', D=D, K=K, weighted=True, ld=D, off=0, B=B, layout='contig', wrap=False)
    if route == 'colmoments':
        _lib.call('elfi_b200_colmoments_f64', dev.context(), S, D, B, D, dev.ptr(mom), dev.stream_ptr())
        c.weighted = False
    else:
        obs = dev.to_device(np.zeros(D))
        W = dev.to_device(np.ones((K, D)))
        d_out = dev.empty((B, K))
        _lib.call('elfi_b200_dist_euclid_mom_f64', dev.context(), S, D, B, D, dev.ptr(obs), dev.ptr(W),
                  K, None, None, dev.ptr(d_out), None, None, dev.ptr(mom), dev.stream_ptr())
    dev.synchronize()
    m = host(mom)
    check_moments(x, m[0], m[1], moments_depth(c, B), '{} {}'.format(route, kind))
    return c


def longdouble_reference_is_exact():
    """The longdouble two-pass reference against exact rational arithmetic on a small batch whose
    first row is far out and whose columns sit on a large offset."""
    rs = np.random.RandomState(11)
    x = rs.randn(40, 5) * 10.0 ** rs.uniform(-3, 3, 5) + 1e6
    x[0] += 1e4
    mean, m2, _, _ = exact_moments(x)
    fm, fm2 = fraction_moments(x)
    tol = 64 * float(np.finfo(np.longdouble).eps)
    for j in range(x.shape[1]):
        em = abs(fractions.Fraction(*mean[j].as_integer_ratio()) - fm[j])
        e2 = abs(fractions.Fraction(*m2[j].as_integer_ratio()) - fm2[j])
        assert em <= tol * abs(fm[j]), (j, float(em))
        assert e2 <= tol * fm2[j], (j, float(e2))
