// philox.cuh -- the counter-based generator of the throughput mode: Philox4x32-10 (Salmon et al.,
// "Parallel random numbers: as easy as 1, 2, 3", SC'11) and its 53-bit uniform on (0, 1].
// Compiles for the host as well (tests/harness/philox_harness.cpp checks it against the
// Random123 known-answer vectors and against the NumPy replay in oracle/streams.py).
#pragma once

#if !defined(__CUDACC_RTC__)   // NVRTC has no C headers: usersim_rt.cuh declares the types
#include <stdint.h>
#endif

#include "hd.cuh"

namespace elfi {

ELFI_HD uint32_t philox_mulhi(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
    return __umulhi(a, b);
#else
    return uint32_t((uint64_t(a) * uint64_t(b)) >> 32);
#endif
}

#if defined(__CUDACC__)
using PhiloxWords = uint4;
#else
struct PhiloxWords { uint32_t x, y, z, w; };
#endif

// key (seed & 0xffffffff, seed >> 32), counter (c0, c1, c2, c3) -> four 32-bit words
struct Philox {
    uint32_t key0, key1;
    ELFI_HD Philox(uint64_t seed) : key0(uint32_t(seed)), key1(uint32_t(seed >> 32)) {}
    ELFI_HD PhiloxWords operator()(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3) const {
        uint32_t k0 = key0, k1 = key1;
#pragma unroll
        for (int r = 0; r < 10; ++r) {
            const uint32_t hi0 = philox_mulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
            const uint32_t hi1 = philox_mulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
            const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
            c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
            k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
        }
        PhiloxWords out;
        out.x = c0; out.y = c1; out.z = c2; out.w = c3;
        return out;
    }
};

// (0, 1] with 53 random bits: the 32 bits of a above the 21 high bits of b, plus one ulp
ELFI_HD double u01(uint32_t a, uint32_t b) {
    const uint64_t v = (uint64_t(a) << 21) ^ uint64_t(b >> 11);
    return (double(v & ((uint64_t(1) << 53) - 1)) + 1.0) * (1.0 / 9007199254740992.0);
}

}  // namespace elfi
