// Host build of elfi_b200/csrc/poisson.cuh (test infrastructure, see tests/test_ricker_host.py).
#include <cstdint>

#include "../../elfi_b200/csrc/poisson.cuh"

// out[i] = log p(k[i]; lam[i])
extern "C" void harness_poisson_logpmf(const double* k, const double* lam, int64_t n, double* out) {
    for (int64_t i = 0; i < n; ++i) out[i] = elfi::poisson_logpmf(k[i], lam[i]);
}

// Draw i from rate lam[i] with the blocks (row, row >> 32, base + j, salt) of Philox(seed), row =
// rows[i]: the count, the blocks used and the smallest decision margin (poisson_draw).
extern "C" void harness_poisson_draw(const double* lam, const uint64_t* rows, int64_t n, uint64_t seed,
                                     uint32_t base, uint32_t salt, double* k, int32_t* trials,
                                     double* margin) {
    const elfi::Philox ph(seed);
    for (int64_t i = 0; i < n; ++i) {
        const uint32_t r0 = uint32_t(rows[i]), r1 = uint32_t(rows[i] >> 32);
        const elfi::PoissonDraw d = elfi::poisson_draw(
            lam[i], [&](int j) { return ph(r0, r1, base + uint32_t(j), salt); });
        k[i] = d.k;
        trials[i] = d.trials;
        margin[i] = d.margin;
    }
}
