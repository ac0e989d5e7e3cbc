// Host build of elfi_b200/csrc/lorenz.cuh (test infrastructure, see tests/test_lorenz_host.py).
#include <cstdint>
#include <vector>

#include "../../elfi_b200/csrc/lorenz.cuh"

// out (T, m): row 0 = init, then T - 1 RK4 steps with forcing eta ((T - 1, m), step s uses row
// s - 1; NULL: eta = 0, the phi = 1 trajectory)
extern "C" void harness_lorenz_run(const double* init, int32_t m, int32_t T, double th1, double th2,
                                   double f, double dt, const double* eta, double* out) {
    std::vector<double> y(init, init + m), zero(m, 0.0), work(5 * m);
    for (int k = 0; k < m; ++k) out[k] = y[k];
    for (int s = 1; s < T; ++s) {
        elfi::lorenz_step_row(y.data(), m, eta ? eta + int64_t(s - 1) * m : zero.data(), dt, f, th1,
                              th2, work.data());
        for (int k = 0; k < m; ++k) out[int64_t(s) * m + k] = y[k];
    }
}

// eta_out (n, m) = lorenz_ar1(eta, e, phi, s) element by element
extern "C" void harness_lorenz_ar1(const double* eta, const double* e, int64_t n, double phi,
                                   double s, double* eta_out) {
    for (int64_t i = 0; i < n; ++i) eta_out[i] = elfi::lorenz_ar1(eta[i], e[i], phi, s);
}

// out (B, 6): the six summaries of the rows x[b * ld_row + t * ld_t + k * ld_k] (T, m)
extern "C" void harness_lorenz_summaries(const double* x, int64_t ld_row, int64_t ld_t,
                                         int64_t ld_k, int64_t B, int32_t T, int32_t m,
                                         double* out) {
    std::vector<double> work(5 * m);
    for (int64_t b = 0; b < B; ++b)
        elfi::lorenz_row_summaries(x + b * ld_row, ld_t, ld_k, T, m, work.data(), out + b * 6);
}
