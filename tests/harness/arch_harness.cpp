// Host build of elfi_b200/csrc/arch.cuh (test infrastructure, see tests/test_arch_host.py).
#include <cmath>
#include <cstdint>

#include "../../elfi_b200/csrc/arch.cuh"

// Y (B, n) = the series of parameters P (B, 2) = (t1, t2) driven by the normals z (B, n + 1):
// z[b, 0] = e_0, z[b, k] = xi_k, as the kernel steps them
extern "C" void harness_arch_rows(const double* P, const double* z, int64_t B, int32_t n,
                                  double* Y) {
    for (int64_t b = 0; b < B; ++b) {
        const double t1 = P[2 * b], t2 = P[2 * b + 1];
        const double* zb = z + b * (n + 1);
        double e = zb[0], y = 0.0;
        for (int k = 1; k <= n; ++k) {
            e = elfi::arch_e(zb[k], e, t2);
            y = elfi::arch_y(t1, y, e);
            Y[b * n + k - 1] = y;
        }
    }
}

// S (B, arch_nsumm(n_lags)) = the summaries of the rows of X (B, n), C-contiguous
extern "C" void harness_arch_summaries(const double* X, int64_t B, int32_t n, int32_t n_lags,
                                       double* S) {
    const int K = elfi::arch_nsumm(n_lags);
    double row[elfi::ARCH_NOBS_MAX];
    for (int64_t b = 0; b < B; ++b) {
        for (int j = 0; j < n; ++j) row[j] = X[b * n + j];
        elfi::arch_summaries(n, n_lags, [&](int j) -> double& { return row[j]; }, S + b * K, 1);
    }
}
