// gnkstats.cuh -- the robust (Drovandi & Pettitt 2011) and octile summaries of the g-and-k
// examples (elfi/examples/gnk.py:164-248) from the sorted observations of one series.
//
// Both summaries are functions of the seven octiles E1..E7 = np.percentile(y, [12.5, 25, ..,
// 87.5]) (L1, L2, L3 = E2, E4, E6), method 'linear' (numpy/lib/_function_base_impl.py, _quantile,
// _get_indexes, _lerp), restated here:
//   vi = (n - 1) * (pct / 100); lo = floor(vi), hi = lo + 1; vi >= n - 1: lo = hi = n - 1 and
//   t = vi + 1 (NumPy keeps the float index against -1, the "last" index), otherwise t = vi - lo;
//   value = t >= 0.5 ? b - (b - a) * (1 - t) : a + (b - a) * t   with a = y[lo], b = y[hi].
//   t == 0 is not a short cut: (inf - a) * 0 is NaN in NumPy too.  A series with a NaN has every
//   percentile NaN (NaN sorts last; NumPy copies the last element).
// The indices and weights depend only on (n, pct) and come from the host (ops.gnk_picks), so the
// device only picks and interpolates.  The epilogue follows gnk.py's order:
//   ss_B = L3 - L1 (+ eps where it is 0), ss_g = ((L3 + L1) - 2 L2) / ss_B,
//   ss_k = (((E7 - E5) + E3) - E1) / ss_B;  robust = [L2, ss_B, ss_g, ss_k], octile = [E1..E7].
// All arithmetic is IEEE round-to-nearest without contraction; the header compiles for the host
// (tests/harness/gnkstats_harness.cpp checks it against NumPy bit for bit).
#pragma once

#include <math.h>

#include "hd.cuh"
#include "leafsum.cuh"

namespace elfi {

constexpr int GNK_NQ = 7;                       // octiles 12.5, 25, .., 87.5 (percent)
constexpr int GNK_ROBUST = 0, GNK_OCTILE = 1;   // summary kinds: 4 or 7 values per dimension

// picks of the seven octiles for one series length: sorted positions lo, hi and weight t
struct GnkPicks {
    int lo[GNK_NQ], hi[GNK_NQ];
    double t[GNK_NQ];
};

ELFI_HD double gnk_div(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}

// numpy _lerp
ELFI_HD double gnk_lerp(double a, double b, double t) {
    const double diff = leaf_sub(b, a);
    return t >= 0.5 ? leaf_sub(b, leaf_mul(diff, leaf_sub(1.0, t))) : leaf_add(a, leaf_mul(diff, t));
}

ELFI_HD int gnk_summary_width(int kind) { return kind == GNK_OCTILE ? GNK_NQ : 4; }

// Octiles from the picked values (a[q] = sorted[lo[q]], b[q] = sorted[hi[q]]) -> the summary of
// one series: out[j * step], j < gnk_summary_width(kind).
ELFI_HD void gnk_summary(int kind, const GnkPicks& p, const double* a, const double* b, bool has_nan,
                         double* out, int step) {
    double E[GNK_NQ];
ELFI_UNROLL
    for (int q = 0; q < GNK_NQ; ++q) E[q] = has_nan ? NAN : gnk_lerp(a[q], b[q], p.t[q]);
    if (kind == GNK_OCTILE) {
ELFI_UNROLL
        for (int q = 0; q < GNK_NQ; ++q) out[q * step] = E[q];
        return;
    }
    const double L1 = E[1], L2 = E[3], L3 = E[5];
    double sB = leaf_sub(L3, L1);
    if (sB == 0.0) sB = leaf_add(sB, 2.220446049250313e-16);   // np.finfo(float).eps
    out[0] = L2;
    out[step] = sB;
    out[2 * step] = gnk_div(leaf_sub(leaf_add(L3, L1), leaf_mul(2.0, L2)), sB);
    out[3 * step] = gnk_div(leaf_sub(leaf_add(leaf_sub(E[6], E[4]), E[2]), E[0]), sB);
}

}  // namespace elfi
