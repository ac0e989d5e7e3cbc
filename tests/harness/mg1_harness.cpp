// Host build of elfi_b200/csrc/mg1.cuh (test infrastructure, see tests/test_mg1_host.py).
#include <cmath>
#include <cstdint>

#include "../../elfi_b200/csrc/mg1.cuh"

// Y (B, n) = the inter-departure times of parameters P (B, 3) = (t1, t2, t3) from the given
// inter-arrival times W (B, n) and service times U (B, n), as the kernel steps them (NaN rows where
// the reference raises)
extern "C" void harness_mg1_rows(const double* P, const double* W, const double* U, int64_t B,
                                 int32_t n, double* Y) {
    for (int64_t b = 0; b < B; ++b) {
        const double inv_t3 = elfi::gnk_div(1.0, P[3 * b + 2]);
        const bool ok = elfi::mg1_params_ok(inv_t3, elfi::leaf_sub(P[3 * b + 1], P[3 * b]));
        double sum_w = 0.0, sum_x = 0.0;
        for (int j = 0; j < n; ++j) {
            const double y = elfi::mg1_step(sum_w, sum_x, W[b * n + j], U[b * n + j]);
            Y[b * n + j] = ok ? y : NAN;
        }
    }
}

// W and U (B, n) from uniforms u, v in (0, 1] as the kernel draws them
extern "C" void harness_mg1_draws(const double* P, const double* u, const double* v, int64_t B,
                                  int32_t n, double* W, double* U) {
    for (int64_t b = 0; b < B; ++b) {
        const double t1 = P[3 * b], t2 = P[3 * b + 1], t3 = P[3 * b + 2];
        for (int j = 0; j < n; ++j) {
            W[b * n + j] = elfi::mg1_gap(elfi::gnk_div(1.0, t3), u[b * n + j]);
            U[b * n + j] = elfi::mg1_service(t1, elfi::leaf_sub(t2, t1), v[b * n + j]);
        }
    }
}

// S (B, nq) = quantiles q of the rows of X (B, n), each row sorted ascending with NaN last
extern "C" void harness_mg1_quantiles(const double* X, int64_t B, int32_t n, const double* q,
                                      int32_t nq, double* S) {
    for (int64_t b = 0; b < B; ++b)
        for (int k = 0; k < nq; ++k)
            S[b * nq + k] = elfi::mg1_quantile(n, q[k], [&](int i) { return X[b * n + i]; });
}
