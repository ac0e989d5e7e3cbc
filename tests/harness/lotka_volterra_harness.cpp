// Host build of elfi_b200/csrc/lotka_volterra.cuh (test infrastructure, see
// tests/test_lotka_volterra_host.py).
#include <cmath>
#include <cstdint>

#include "../../elfi_b200/csrc/lotka_volterra.cuh"

// Runs one row of parameters p (6) as the kernel does, with the event draws E[k], u[k]
// (k < max_events) and the observation normals z[2 j], z[2 j + 1] given: obs (n_obs, 2), returns
// the number of events.  NaN observations where the kernel writes them.
extern "C" int64_t harness_lv_row(const double* p, const double* E, const double* u,
                                  const double* z, const double* t_out, int32_t n_obs,
                                  double time_end, int64_t max_events, double* obs) {
    elfi::LvState s;
    bool ok = elfi::lv_init(s, p);
    if (ok) {
        obs[0] = s.X;
        obs[1] = s.Y;
        while (ok && elfi::lv_running(s, time_end, uint32_t(max_events)))
            ok = elfi::lv_advance(
                s, E[s.k], u[s.k], t_out, n_obs, time_end,
                [&](int j, double& n0, double& n1) {
                    n0 = z[2 * j];
                    n1 = z[2 * j + 1];
                },
                [&](int j, double prey, double pred) {
                    obs[2 * j] = prey;
                    obs[2 * j + 1] = pred;
                });
        ok = ok && elfi::lv_complete(s, time_end, n_obs);
    }
    if (!ok)
        for (int i = 0; i < 2 * n_obs; ++i) obs[i] = NAN;
    return s.k;
}

// out[i] = the int32 truncation of v[i] (as a double)
extern "C" void harness_lv_to_int32(const double* v, int64_t n, double* out) {
    for (int64_t i = 0; i < n; ++i) out[i] = elfi::lv_to_int32(v[i]);
}

// S (B, 9) = the nine summaries of X (B, n, 2), C-contiguous
extern "C" void harness_lv_summaries(const double* X, int64_t B, int32_t n, double* S) {
    for (int64_t b = 0; b < B; ++b) {
        const double* x = X + b * 2 * n;
        elfi::lv_summaries(n, [&](int i, int sp) { return x[2 * i + sp]; }, S + b * 9);
    }
}
