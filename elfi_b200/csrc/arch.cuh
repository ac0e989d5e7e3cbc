// arch.cuh -- the arithmetic of the ARCH(1) model of elfi/examples/arch.py, shared by the device
// kernels (arch.cu) and the host build of the tests (tests/harness/arch_harness.cpp, g++
// -ffp-contract=off): the recurrence step and the 2 + L + L(L-1)/2 summaries of one row.
//
// Every operation is rounded on its own, in the reference's order (arch.py:100-132):
//   e_i = xi_i * sqrt(0.2 + t2 * (e_{i-1} * e_{i-1})),   y_i = t1 * y_{i-1} + e_i,   y_0 = 0.
// The summaries follow NumPy (arch.py:135-208).  Rows have 2 <= n <= 128 observations, so every
// reduction is one leaf of NumPy's pairwise sum (LeafSum):
//   MU  = (0.0 + pairwise(y)) / n
//   VAR = pairwise((y - MU)^2) / (n - 1)                      (np.var, ddof = 1)
//   sc  = (y - MU) / sqrt(VAR)                                (autocorr's np.mean / np.std: same bits)
//   AC_lag = pairwise(sc[j + lag] * sc[j], j < n - lag) / (n - lag),  lag = 1 .. L
//   PW_i_j = AC_i * AC_j   for (i, j) in itertools.combinations(range(1, L + 1), 2)
// +, -, *, / and sqrt are correctly rounded on both sides, so the device equals NumPy bit for bit.
#pragma once

#include <math.h>
#include <stdint.h>

#include "hd.cuh"
#include "../../include/elfi_b200.h"
#include "leafsum.cuh"

namespace elfi {

constexpr int ARCH_NOBS_MIN = ELFI_B200_ARCH_NOBS_MIN;
constexpr int ARCH_NOBS_MAX = ELFI_B200_ARCH_NOBS_MAX;
static_assert(ARCH_NOBS_MAX == LEAF_MAX_TERMS, "one pairwise leaf per reduction");
constexpr int ARCH_LAGS_MAX = ELFI_B200_ARCH_LAGS_MAX;

ELFI_HD double arch_div(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}
ELFI_HD double arch_sqrt(double a) {
#if defined(__CUDA_ARCH__)
    return __dsqrt_rn(a);
#else
    return sqrt(a);
#endif
}

ELFI_HD int arch_nsumm(int n_lags) { return 2 + n_lags + n_lags * (n_lags - 1) / 2; }

// e_i from xi_i and e_{i-1}: xi * sqrt(0.2 + t2 * e^2), np.power(e, 2) being e * e
ELFI_HD double arch_e(double xi, double e_prev, double t2) {
    return leaf_mul(xi, arch_sqrt(leaf_add(0.2, leaf_mul(t2, leaf_mul(e_prev, e_prev)))));
}
// y_i = t1 * y_{i-1} + e_i
ELFI_HD double arch_y(double t1, double y_prev, double e) { return leaf_add(leaf_mul(t1, y_prev), e); }

template <int J, class F>
ELFI_HD void arch_push8(LeafSum& s, int j0, int m, const F& term) {
    const int j = j0 + J;
    if (j < m) s.push<J>(j, term(j));
    if constexpr (J + 1 < 8) arch_push8<J + 1>(s, j0, m, term);
}

// np.add.reduce of term(0 .. m-1), 1 <= m <= 128
template <class F>
ELFI_HD double arch_sum(int m, const F& term) {
    LeafSum s;
    s.begin(m);
    for (int j0 = 0; j0 < m; j0 += 8) arch_push8<0>(s, j0, m, term);
    return s.finish(m);
}

// The summaries of one row.  x(j) returns a reference to observation j (0 <= j < n); the row is
// overwritten by its standardised values sc.  out[k * ld], k < arch_nsumm(n_lags), in the order
// MU, VAR, AC_1 .. AC_L, PW in combinations order.
template <class Row>
ELFI_HD void arch_summaries(int n, int n_lags, const Row& x, double* out, int64_t ld) {
    const double mean = arch_div(arch_sum(n, [&](int j) { return x(j); }), double(n));
    const double var = arch_div(arch_sum(n, [&](int j) {
                                    const double c = leaf_sub(x(j), mean);
                                    return leaf_mul(c, c);
                                }),
                                double(n - 1));
    const double sd = arch_sqrt(var);
    for (int j = 0; j < n; ++j) x(j) = arch_div(leaf_sub(x(j), mean), sd);
    out[0] = mean;
    out[ld] = var;
    double ac[ARCH_LAGS_MAX];
ELFI_UNROLL
    for (int lag = 1; lag <= ARCH_LAGS_MAX; ++lag) {
        ac[lag - 1] = 0.0;
        if (lag > n_lags) continue;
        ac[lag - 1] = arch_div(arch_sum(n - lag, [&](int j) { return leaf_mul(x(j + lag), x(j)); }),
                               double(n - lag));
        out[(1 + lag) * ld] = ac[lag - 1];
    }
    int k = 2 + n_lags;
ELFI_UNROLL
    for (int i = 0; i < ARCH_LAGS_MAX; ++i) {
ELFI_UNROLL
        for (int j = i + 1; j < ARCH_LAGS_MAX; ++j) {
            if (j < n_lags) {
                out[k * ld] = leaf_mul(ac[i], ac[j]);
                ++k;
            }
        }
    }
}

}  // namespace elfi
