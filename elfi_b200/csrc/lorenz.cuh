// lorenz.cuh -- arithmetic of the Lorenz forecast model (elfi/examples/lorenz.py; Wilks 2005): the
// derivative, the RK4 step and the AR(1) forcing in the reference's order of operations, and the
// pieces of its six summaries in NumPy's summation orders.  Every operation is rounded on its own
// (no FMA): leaf_add / leaf_sub / leaf_mul and lorenz_div are __dadd_rn & co. on the device and
// plain operators on the host, where tests/harness/lorenz_harness.cpp builds this header with
// -ffp-contract=off and checks it against NumPy bit for bit.
//
// Summaries of one row x (T, m), as the reference computes them on a C-contiguous (B, T, m) array:
//   column sums   np.mean / np.var(x, axis=1) and the means of x[:, :-1] / x[:, 1:] add the rows
//                 one after the other, from 0.0: S_A[k] = sum_{t < T-1} x[t, k], S_B[k] =
//                 sum_{t >= 1} x[t, k], and the sum over all t is S_A[k] + x[T-1, k];
//   flat sums     np.mean(., axis=(1, 2)) and np.mean(., axis=1) of a (B, m) result are NumPy's
//                 pairwise sum over the flattened row (t-major, k-minor): leaves of at most 128
//                 terms (8 strided accumulators, a fold, a sequential tail), longer runs split at
//                 n / 2 rounded down to a multiple of 8, left part first; 0.0 + the total.
// PairwiseLeaves walks the leaves of such a sum in order and combines their values; the caller
// computes each leaf (lorenz_leaf_value here, an 8-lane group on the device).
#pragma once

#include <stdint.h>

#include "hd.cuh"
#include "../../include/elfi_b200.h"
#include "leafsum.cuh"

namespace elfi {

constexpr int LORENZ_SUMM_MAXD = 8;   // open splits of PairwiseLeaves
// longest flattened run PairwiseLeaves takes (TreeSum's bound: a right part has up to n/2 + 7
// terms); the summaries need n_timestep * n_obs <= this
constexpr int64_t LORENZ_SUMM_MAX_TERMS = ELFI_B200_LORENZ_SUMM_MAX_TERMS;
static_assert(LORENZ_SUMM_MAX_TERMS == (int64_t(120) << LORENZ_SUMM_MAXD) + 8,
              "the summaries' bound is the longest run PairwiseLeaves takes");

ELFI_HD double lorenz_div(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}

// dy_k/dt of _lorenz_ode, left to right:
//   -y[k-2] * y[k-1] + y[k-1] * y[k+1] - y[k] + f - (theta1 + y[k] * theta2) + eta[k]
ELFI_HD double lorenz_deriv(double ym2, double ym1, double y, double yp1, double f, double th1,
                            double th2, double eta) {
    const double g = leaf_add(th1, leaf_mul(y, th2));
    double d = leaf_add(leaf_mul(-ym2, ym1), leaf_mul(ym1, yp1));
    d = leaf_sub(d, y);
    d = leaf_add(d, f);
    d = leaf_sub(d, g);
    return leaf_add(d, eta);
}

// runge_kutta_ode_solver: k_j = dt * ode(stage_j); stages y + k1 / 2, y + k2 / 2, y + k3 (k / 2 is
// k * 0.5: both exact); y + (k1 + 2 k2 + 2 k3 + k4) / 6 with a real division by 6
ELFI_HD double lorenz_half_stage(double y, double k) { return leaf_add(y, leaf_mul(k, 0.5)); }
ELFI_HD double lorenz_update(double y, double k1, double k2, double k3, double k4) {
    const double s = leaf_add(leaf_add(leaf_add(k1, leaf_mul(2.0, k2)), leaf_mul(2.0, k3)), k4);
    return leaf_add(y, lorenz_div(s, 6.0));
}

// eta = phi * eta + e * sqrt(1 - phi^2); s = sqrt(1 - phi^2) comes from the host, computed as the
// reference computes it (phi > 1 makes it NaN)
ELFI_HD double lorenz_ar1(double eta, double e, double phi, double s) {
    return leaf_add(leaf_mul(phi, eta), leaf_mul(e, s));
}

// (x[t, k] - a) * (x[t + 1, k'] - b): the terms of Autocov and the two Crosscov summaries
ELFI_HD double lorenz_cross(double x0, double a, double x1, double b) {
    return leaf_mul(leaf_sub(x0, a), leaf_sub(x1, b));
}

// The leaves of NumPy's pairwise sum of n terms, in order, and the sum of their values.
//   begin(n); do { v = value of leaf [start, start + len); } while (add_leaf(v));  total()
template <int MAXD>
struct PairwiseLeaves {
    double left_val[MAXD];     // [0] = innermost open split
    int pending_right[MAXD];   // length of the right part still to come, per open split
    uint32_t has_left;         // bit d: split d already holds its left sum
    int depth;
    int start, len;            // the current leaf
    double sum;

    ELFI_HD void open_split(int right) {
ELFI_UNROLL
        for (int d = MAXD - 1; d > 0; --d) {
            pending_right[d] = pending_right[d - 1];
            left_val[d] = left_val[d - 1];
        }
        pending_right[0] = right;
        left_val[0] = 0.0;
        has_left <<= 1;
        ++depth;
    }
    ELFI_HD void close_split() {
ELFI_UNROLL
        for (int d = 0; d < MAXD - 1; ++d) {
            pending_right[d] = pending_right[d + 1];
            left_val[d] = left_val[d + 1];
        }
        has_left >>= 1;
        --depth;
    }
    ELFI_HD void descend(int s, int n) {
        while (n > LEAF_MAX_TERMS) {
            int left = n / 2;
            left -= left % 8;
            open_split(n - left);
            n = left;
        }
        start = s;
        len = n;
    }
    ELFI_HD void begin(int n) {
        depth = 0;
        has_left = 0;
        sum = 0.0;
ELFI_UNROLL
        for (int d = 0; d < MAXD; ++d) {
            left_val[d] = 0.0;
            pending_right[d] = 0;
        }
        descend(0, n);
    }
    // hands the current leaf's value up the open splits; false after the last leaf
    ELFI_HD bool add_leaf(double v) {
        const int next = start + len;
        while (depth > 0) {
            if (!(has_left & 1u)) {
                left_val[0] = v;
                has_left |= 1u;
                descend(next, pending_right[0]);
                return true;
            }
            v = leaf_add(left_val[0], v);
            close_split();
        }
        sum = v;
        return false;
    }
    // np.add.reduce starts from the identity (see LeafSum::finish)
    ELFI_HD double total() const { return leaf_add(0.0, sum); }
};

// the fold of a leaf's 8 accumulators
ELFI_HD double lorenz_fold(const double* r) {
    return leaf_add(leaf_add(leaf_add(r[0], r[1]), leaf_add(r[2], r[3])),
                    leaf_add(leaf_add(r[4], r[5]), leaf_add(r[6], r[7])));
}

// value of the leaf [s, s + L) of term(j), serially (the host's form of the device's 8-lane leaf)
template <class Term>
inline double lorenz_leaf_value(int s, int L, const Term& term) {
    if (L < 8) {
        double res = 0.0;
        for (int i = 0; i < L; ++i) res = leaf_add(res, term(s + i));
        return res;
    }
    const int L8 = L - L % 8;
    double r[8];
    for (int c = 0; c < 8; ++c) r[c] = term(s + c);
    for (int i = 8; i < L8; i += 8)
        for (int c = 0; c < 8; ++c) r[c] = leaf_add(r[c], term(s + i + c));
    double res = lorenz_fold(r);
    for (int i = L8; i < L; ++i) res = leaf_add(res, term(s + i));
    return res;
}

template <class Term>
inline double lorenz_pairwise(int n, const Term& term) {
    PairwiseLeaves<LORENZ_SUMM_MAXD> w;
    w.begin(n);
    while (w.add_leaf(lorenz_leaf_value(w.start, w.len, term))) {
    }
    return w.total();
}

// Host form of the six summaries [Mean, Var, Autocov, Cov, CrosscovPrev, CrosscovNext] of one row
// x[t * ldt + k * ldk], 2 <= T, 2 <= m <= 128 (for m = 1 NumPy sums over time pairwise), T * m <= LORENZ_SUMM_MAX_TERMS.  work: 5 * m doubles.
inline void lorenz_row_summaries(const double* x, int64_t ldt, int64_t ldk, int T, int m,
                                 double* work, double* out) {
    double* M = work;          // mean over all t
    double* A = work + m;      // mean over t < T - 1
    double* Bm = work + 2 * m; // mean over t >= 1
    double* V = work + 3 * m;  // np.var over t
    double* C = work + 4 * m;  // covariance with column k + 1 over t
    auto X = [&](int t, int k) { return x[t * ldt + k * ldk]; };
    for (int k = 0; k < m; ++k) {
        double sa = 0.0, sb = 0.0;
        for (int t = 0; t < T - 1; ++t) {
            sa = leaf_add(sa, X(t, k));
            sb = leaf_add(sb, X(t + 1, k));
        }
        M[k] = lorenz_div(leaf_add(sa, X(T - 1, k)), double(T));
        A[k] = lorenz_div(sa, double(T - 1));
        Bm[k] = lorenz_div(sb, double(T - 1));
    }
    for (int k = 0; k < m; ++k) {
        const int kr = (k + 1 == m) ? 0 : k + 1;
        double v = 0.0, c = 0.0;
        for (int t = 0; t < T; ++t) {
            const double d = leaf_sub(X(t, k), M[k]);
            v = leaf_add(v, leaf_mul(d, d));
            c = leaf_add(c, leaf_mul(d, leaf_sub(X(t, kr), M[kr])));
        }
        V[k] = lorenz_div(v, double(T));
        C[k] = lorenz_div(c, double(T));
    }
    const int n1 = (T - 1) * m;
    out[0] = lorenz_div(lorenz_pairwise(T * m, [&](int j) { return X(j / m, j % m); }),
                        double(T * m));
    out[1] = lorenz_div(lorenz_pairwise(m, [&](int k) { return V[k]; }), double(m));
    out[2] = lorenz_div(lorenz_pairwise(n1, [&](int j) {
                            const int t = j / m, k = j % m;
                            return lorenz_cross(X(t, k), A[k], X(t + 1, k), Bm[k]);
                        }), double(n1));
    out[3] = lorenz_div(lorenz_pairwise(m, [&](int k) { return C[k]; }), double(m));
    out[4] = lorenz_div(lorenz_pairwise(n1, [&](int j) {
                            const int t = j / m, k = j % m, kl = (k == 0) ? m - 1 : k - 1;
                            return lorenz_cross(X(t, k), A[k], X(t + 1, kl), Bm[kl]);
                        }), double(n1));
    out[5] = lorenz_div(lorenz_pairwise(n1, [&](int j) {
                            const int t = j / m, k = j % m, kr = (k + 1 == m) ? 0 : k + 1;
                            return lorenz_cross(X(t, k), A[k], X(t + 1, kr), Bm[kr]);
                        }), double(n1));
}

// Host form of one RK4 step of a whole row y (m) with forcing eta (m); work: 5 * m doubles
inline void lorenz_step_row(double* y, int m, const double* eta, double dt, double f, double th1,
                            double th2, double* work) {
    double* k1 = work;
    double* k2 = work + m;
    double* k3 = work + 2 * m;
    double* k4 = work + 3 * m;
    double* st = work + 4 * m;
    auto ode = [&](const double* s, double* kout) {
        for (int k = 0; k < m; ++k) {
            const int km2 = (k + m - 2) % m, km1 = (k + m - 1) % m, kp1 = (k + 1) % m;
            kout[k] = leaf_mul(dt, lorenz_deriv(s[km2], s[km1], s[k], s[kp1], f, th1, th2, eta[k]));
        }
    };
    ode(y, k1);
    for (int k = 0; k < m; ++k) st[k] = lorenz_half_stage(y[k], k1[k]);
    ode(st, k2);
    for (int k = 0; k < m; ++k) st[k] = lorenz_half_stage(y[k], k2[k]);
    ode(st, k3);
    for (int k = 0; k < m; ++k) st[k] = leaf_add(y[k], k3[k]);
    ode(st, k4);
    for (int k = 0; k < m; ++k) y[k] = lorenz_update(y[k], k1[k], k2[k], k3[k], k4[k]);
}

}  // namespace elfi
