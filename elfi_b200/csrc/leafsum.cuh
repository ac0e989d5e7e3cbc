// leafsum.cuh -- single-leaf form of NumPy's pairwise summation for rows of <= 128 terms.
//
// For a run of m <= 128 terms DOUBLE_pairwise_sum does not recurse: m < 8 is a plain
// left-to-right sum starting from 0.0; otherwise r[k] = a[k] (k < 8), r[k] += a[8i + k] for the
// whole groups, res = ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), and the m % 8 trailing terms are added
// to res one by one.  That is all the state the benchmark shapes need (MA2: 99 / 98 products per
// row, Gaussian model: 50 observations; elfi/examples/ma2.py:40-59, gauss.py:142-173), so the
// row-stream summary kernels use this instead of the general PairwiseStream tree whenever every
// reduced run fits one leaf: no stack, no per-group state machine, and column groups whose 16
// terms all fall in the "whole groups" range take a branch-free path.
//
// The arithmetic lives in plain structs that also compile for the host (tests/harness builds
// them with g++ -ffp-contract=off and checks them against NumPy bit for bit); the device
// kernels in summaries.cu only add the shared-memory read of the 16 columns.
#pragma once

#include "hd.cuh"

namespace elfi {

ELFI_HD double leaf_add(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
ELFI_HD double leaf_sub(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dsub_rn(a, b);
#else
    return a - b;
#endif
}
ELFI_HD double leaf_mul(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}

constexpr int LEAF_MAX_TERMS = 128;   // NumPy's PW_BLOCKSIZE
constexpr int LEAF_BOX = 16;          // columns handed over per call (one TMA box row)

// Terms are pushed strictly in index order; K = j % 8 is a compile-time constant at every
// call site so r[] stays in registers.
struct LeafSum {
    double r[8];
    double res;
    int m8;   // index of the first tail term: m - m % 8, or 0 when m < 8 (everything is tail)

    ELFI_HD void begin(int m) {
        m8 = (m < 8) ? 0 : (m & ~7);
        res = 0.0;
ELFI_UNROLL
        for (int k = 0; k < 8; ++k) r[k] = 0.0;
    }
    ELFI_HD double fold() const {
        return leaf_add(leaf_add(leaf_add(r[0], r[1]), leaf_add(r[2], r[3])),
                        leaf_add(leaf_add(r[4], r[5]), leaf_add(r[6], r[7])));
    }
    // any term 0 <= j < m
    template <int K>
    ELFI_HD void push(int j, double v) {
        if (j >= m8) {
            if (j == m8 && m8 > 0) res = fold();
            res = leaf_add(res, v);
        } else if (j < 8) {
            r[K] = v;
        } else {
            r[K] = leaf_add(r[K], v);
        }
    }
    // a term known to satisfy 8 <= j < m8
    template <int K>
    ELFI_HD void push_mid(double v) {
        r[K] = leaf_add(r[K], v);
    }
    ELFI_HD bool all_mid(int j_first, int j_last) const { return j_first >= 8 && j_last < m8; }
    // np.add.reduce starts from the identity: the result is 0.0 + pairwise_sum, which only
    // matters for the sign of a zero sum (-0.0 becomes +0.0)
    ELFI_HD double finish(int m) const {
        return leaf_add(0.0, (m >= 8 && (m & 7) == 0) ? fold() : res);
    }
};

// The box feeders below are templates over the accumulator `Sum` (LeafSum here, TreeSum in
// treesum.cuh): begin(m), push<K>(j, v), push_mid<K>(v), all_mid(j_first, j_last), finish(m).

// sum_j x[j + LAG] * x[j], j = 0 .. n-LAG-1, for one or two lags, fed 16 columns at a time.
// LAG_B = -1 disables the second lag.  Lags are at most 8 so the previous box's tail fits hist[].
template <class Sum, int LAG_A, int LAG_B>
struct AutocovBoxes {
    static constexpr int HMAX = (LAG_A > LAG_B ? LAG_A : LAG_B);
    Sum sa, sb;
    double hist[HMAX];   // last HMAX columns of the previous box
    int n;

    ELFI_HD void begin(int n_) {
        n = n_;
        sa.begin(n - LAG_A);
        if (LAG_B >= 0) sb.begin(n - LAG_B);
ELFI_UNROLL
        for (int h = 0; h < HMAX; ++h) hist[h] = 0.0;
    }
    template <int LAG, int C>
    ELFI_HD double product(const double* cur) const {
        const double prev = (C >= LAG) ? cur[C >= LAG ? C - LAG : 0]
                                       : hist[C >= LAG ? 0 : HMAX - LAG + C];
        return leaf_mul(cur[C], prev);
    }
    template <int LAG, int C>
    ELFI_HD void steps(Sum& s, int t0, const double* cur) {
        const int t = t0 + C;   // element index; product index j = t - LAG
        if (t >= LAG && t < n) s.template push<((C - LAG) % 8 + 8) % 8>(t - LAG, product<LAG, C>(cur));
        if constexpr (C + 1 < LEAF_BOX) steps<LAG, C + 1>(s, t0, cur);
    }
    template <int LAG, int C>
    ELFI_HD void steps_mid(Sum& s, const double* cur) {
        s.template push_mid<((C - LAG) % 8 + 8) % 8>(product<LAG, C>(cur));
        if constexpr (C + 1 < LEAF_BOX) steps_mid<LAG, C + 1>(s, cur);
    }
    template <int LAG>
    ELFI_HD void lag_box(Sum& s, int t0, const double* cur) {
        if (s.all_mid(t0 - LAG, t0 + LEAF_BOX - 1 - LAG))
            steps_mid<LAG, 0>(s, cur);
        else
            steps<LAG, 0>(s, t0, cur);
    }
    // cur[c] = x[t0 + c]; columns at or beyond n are never read into a term
    ELFI_HD void box(int t0, const double* cur) {
        lag_box<LAG_A>(sa, t0, cur);
        if constexpr (LAG_B >= 0) lag_box<LAG_B>(sb, t0, cur);
ELFI_UNROLL
        for (int h = 0; h < HMAX; ++h) hist[h] = cur[LEAF_BOX - HMAX + h];
    }
    ELFI_HD double sum_a() const { return sa.finish(n - LAG_A); }
    ELFI_HD double sum_b() const { return sb.finish(n - LAG_B); }
};

template <int LAG_A, int LAG_B>
using AutocovLeaf = AutocovBoxes<LeafSum, LAG_A, LAG_B>;

// Row mean and (population) variance in two sweeps over the same boxes:
// sweep 0 sums x, sweep 1 sums (x - mean)^2   (numpy _mean / _var, ddof = 0).
template <class Sum>
struct MeanVarBoxes {
    Sum s;
    double mean;
    int n;

    ELFI_HD void begin(int n_) {
        n = n_;
        mean = 0.0;
        s.begin(n);
    }
    template <int C>
    ELFI_HD double value(int pass, const double* cur) const {
        if (pass == 0) return cur[C];
        const double c = leaf_sub(cur[C], mean);
        return leaf_mul(c, c);
    }
    template <int C>
    ELFI_HD void steps(int pass, int t0, const double* cur) {
        if (t0 + C < n) s.template push<C % 8>(t0 + C, value<C>(pass, cur));
        if constexpr (C + 1 < LEAF_BOX) steps<C + 1>(pass, t0, cur);
    }
    template <int C>
    ELFI_HD void steps_mid(int pass, const double* cur) {
        s.template push_mid<C % 8>(value<C>(pass, cur));
        if constexpr (C + 1 < LEAF_BOX) steps_mid<C + 1>(pass, cur);
    }
    ELFI_HD void box(int pass, int t0, const double* cur) {
        if (pass == 1 && t0 == 0) {   // first box of the second sweep: close the mean
            mean = s.finish(n) / double(n);
            s.begin(n);
        }
        if (s.all_mid(t0, t0 + LEAF_BOX - 1))
            steps_mid<0>(pass, cur);
        else
            steps<0>(pass, t0, cur);
    }
    ELFI_HD double variance() const { return s.finish(n) / double(n); }
};

using MeanVarLeaf = MeanVarBoxes<LeafSum>;

// Row mean and variance from ONE sweep for rows of <= 16 * NBOX <= 64 observations (the Gaussian
// model has 50): the row is kept in registers while the boxes go by, so the variance terms
// (x - mean)^2 are formed from registers instead of a second sweep over the boxes.  Same
// LeafSum order as MeanVarBoxes, hence the same bits.  G (the box index) is a compile-time
// constant at every call site so that x[] stays in registers.
template <int NBOX>
struct MeanVarRegs {
    LeafSum s;
    double x[NBOX * LEAF_BOX];
    int n;

    ELFI_HD void begin(int n_) {
        n = n_;
        s.begin(n);
    }
    template <int G, int C>
    ELFI_HD void keep(const double* cur) {
        x[G * LEAF_BOX + C] = cur[C];
        if (G * LEAF_BOX + C < n) s.template push<C % 8>(G * LEAF_BOX + C, cur[C]);
        if constexpr (C + 1 < LEAF_BOX) keep<G, C + 1>(cur);
    }
    template <int G, int C>
    ELFI_HD void keep_mid(const double* cur) {
        x[G * LEAF_BOX + C] = cur[C];
        s.template push_mid<C % 8>(cur[C]);
        if constexpr (C + 1 < LEAF_BOX) keep_mid<G, C + 1>(cur);
    }
    template <int G>
    ELFI_HD void box(const double* cur) {
        if (s.all_mid(G * LEAF_BOX, G * LEAF_BOX + LEAF_BOX - 1))
            keep_mid<G, 0>(cur);
        else
            keep<G, 0>(cur);
    }
    template <int J>
    ELFI_HD void squares(double mean) {
        if (J < n) {
            const double c = leaf_sub(x[J], mean);
            s.template push<J % 8>(J, leaf_mul(c, c));
        }
        if constexpr (J + 1 < NBOX * LEAF_BOX) squares<J + 1>(mean);
    }
    // after the last box: mean and variance of the row
    ELFI_HD void finish(double& mean, double& var) {
        mean = s.finish(n) / double(n);
        s.begin(n);
        squares<0>(mean);
        var = s.finish(n) / double(n);
    }
};

}  // namespace elfi
