// Host build of elfi_b200/csrc/ar1.cuh (test infrastructure, see tests/test_ar1_host.py).
#include <cmath>
#include <cstdint>

#include "../../elfi_b200/csrc/ar1.cuh"

// X (B, n) = the series of parameters phi (B) driven by the innovations w (B, n), w[b, t] being
// the innovation of observation t + 1, as the kernel steps them; d (B) = the distance of each
// series to y (n), accumulated step by step as the kernel does it (d may be NULL)
extern "C" void harness_ar1_rows(const double* phi, const double* w, int64_t B, int32_t n,
                                 const double* y, double* X, double* d) {
    for (int64_t b = 0; b < B; ++b) {
        double x = 0.0, acc = 0.0;
        for (int t = 0; t < n; ++t) {
            x = elfi::ar1_step(phi[b], x, w[b * n + t]);
            X[b * n + t] = x;
            if (d) acc = elfi::ar1_dist_term(acc, x, y[t]);
        }
        if (d) d[b] = elfi::ar1_dist_finish(acc);
    }
}
