// Host build of the CUDA toolkit's own Philox4x32-10 (curand_philox4x32_x.h), an implementation
// independent of this project's, to pin the NumPy replay of oracle/streams.py (test
// infrastructure, see tests/test_streams_host.py; compiled by nvcc, run on the CPU).
#include <cstdint>

#define QUALIFIERS static inline __host__ __device__
#include <curand_philox4x32_x.h>

// ctr: n x 4 counter words, key: n x 2 key words; out: n x 4 output words
extern "C" void harness_curand_philox(const uint32_t* ctr, const uint32_t* key, int64_t n,
                                      uint32_t* out) {
    for (int64_t i = 0; i < n; ++i) {
        const uint4 c = make_uint4(ctr[4 * i], ctr[4 * i + 1], ctr[4 * i + 2], ctr[4 * i + 3]);
        const uint2 k = make_uint2(key[2 * i], key[2 * i + 1]);
        const uint4 r = curand_Philox4x32_10(c, k);
        out[4 * i] = r.x;
        out[4 * i + 1] = r.y;
        out[4 * i + 2] = r.z;
        out[4 * i + 3] = r.w;
    }
}
