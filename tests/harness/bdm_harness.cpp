// Host build of elfi_b200/csrc/bdm.cuh (test infrastructure, see tests/test_bdm_host.py).
#include <cmath>
#include <cstdint>
#include <random>
#include <vector>

#include "../../elfi_b200/csrc/bdm.cuh"

// The rows of P (B, 4: alpha, delta, tau, N) driven as the reference executable drives them: one
// std::mt19937(seed) across the rows, std::uniform_real_distribution<double>(0, 1), u then v per
// event.  out[i * ld + j] = count j of row i (j < N of the row).  Returns 0, or -1 for a row whose
// rates bdm_init refuses.
extern "C" int harness_bdm_mt(const double* P, int64_t B, uint32_t seed, uint32_t* out,
                              int64_t ld) {
    std::mt19937 gen(seed);
    std::uniform_real_distribution<double> unif(0.0, 1.0);
    for (int64_t i = 0; i < B; ++i) {
        const double* p = P + 4 * i;
        const int N = int(p[3]);
        std::vector<uint16_t> c(N);
        elfi::BdmState s;
        if (!elfi::bdm_init(s, p[0], p[1], p[2], N, c.data(), 1)) return -1;
        while (elfi::bdm_running(s)) {
            const double u = unif(gen);
            const double v = unif(gen);
            elfi::bdm_step(s, u, v, c.data(), 1);
        }
        elfi::bdm_finish(s, c.data(), 1);
        for (int j = 0; j < N; ++j) out[i * ld + j] = c[j];
    }
    return 0;
}

// One row per parameter row of P (B, 3) with population bound N, run as the kernel runs it from
// the given uniforms u[i * ldU + k], v[i * ldU + k] (k < ldU): X (B, N) counts and n_events, with
// the kernel's -1 counts for invalid (n_events = -1) and capped (n_events = max_events) rows.
extern "C" void harness_bdm_rows(const double* P, int64_t B, int32_t N, const double* u,
                                 const double* v, int64_t ldU, int64_t max_events, int16_t* X,
                                 int64_t* n_events) {
    std::vector<uint16_t> c(N);
    for (int64_t i = 0; i < B; ++i) {
        elfi::BdmState s;
        int16_t* x = X + i * N;
        if (!elfi::bdm_init(s, P[3 * i], P[3 * i + 1], P[3 * i + 2], N, c.data(), 1)) {
            for (int j = 0; j < N; ++j) x[j] = -1;
            n_events[i] = -1;
            continue;
        }
        while (elfi::bdm_running(s) && int64_t(s.k) < max_events && int64_t(s.k) < ldU)
            elfi::bdm_step(s, u[i * ldU + s.k], v[i * ldU + s.k], c.data(), 1);
        const bool done = !elfi::bdm_running(s);
        if (done) elfi::bdm_finish(s, c.data(), 1);
        for (int j = 0; j < N; ++j) x[j] = done ? int16_t(c[j]) : int16_t(-1);
        n_events[i] = s.k;
    }
}

// S (B, 2) = T1, T2 (with n) of X (B, N), C-contiguous
extern "C" void harness_bdm_summaries(const int16_t* X, int64_t B, int32_t N, double n,
                                      double* S) {
    for (int64_t b = 0; b < B; ++b) {
        const int16_t* x = X + b * N;
        elfi::bdm_summaries(N, n, [&](int j) { return x[j]; }, S + 2 * b);
    }
}
