// Host build of elfi_b200/csrc/philox.cuh (test infrastructure, see tests/test_streams_host.py).
#include <cstdint>

#include "../../elfi_b200/csrc/philox.cuh"

// ctr: n x 4 counter words, seed: n keys; out: n x 4 output words
extern "C" void harness_philox(const uint32_t* ctr, const uint64_t* seed, int64_t n, uint32_t* out) {
    for (int64_t i = 0; i < n; ++i) {
        const elfi::PhiloxWords r = elfi::Philox(seed[i])(ctr[4 * i], ctr[4 * i + 1], ctr[4 * i + 2],
                                                          ctr[4 * i + 3]);
        out[4 * i] = r.x;
        out[4 * i + 1] = r.y;
        out[4 * i + 2] = r.z;
        out[4 * i + 3] = r.w;
    }
}

extern "C" void harness_u01(const uint32_t* a, const uint32_t* b, int64_t n, double* out) {
    for (int64_t i = 0; i < n; ++i) out[i] = elfi::u01(a[i], b[i]);
}
