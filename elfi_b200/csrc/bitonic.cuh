// bitonic.cuh -- per-row sorting networks shared by the row sort (select.cu, np.sort(y, axis=1))
// and the g-and-k order-statistic summaries (gnkstats.cu).  Keys are fp64 mapped to
// order-preserving u64 (NaN last, like NumPy); ~0 is both NaN and the padding of a row.
#pragma once

#include <stdint.h>

namespace elfi {

__device__ __forceinline__ uint64_t key_to_u64(double d) {
    if (d != d) return ~uint64_t(0);                 // NaN sorts last
    uint64_t u = static_cast<uint64_t>(__double_as_longlong(d));
    return (u >> 63) ? ~u : (u | (uint64_t(1) << 63));
}
__device__ __forceinline__ double u64_to_key(uint64_t u) {
    if (u == ~uint64_t(0)) return __longlong_as_double(0x7ff8000000000000LL);
    u = (u >> 63) ? (u & ~(uint64_t(1) << 63)) : ~u;
    return __longlong_as_double(static_cast<long long>(u));
}

// The network on npow2 (a power of two) keys in shared memory, ascending: nt threads (this one
// is t0) share the npow2 / 2 compare-exchanges of a stage, and Sync::wait() separates stages.
template <class Sync>
__device__ __forceinline__ void bitonic_network_shared(uint64_t* sk, int npow2, int t0, int nt) {
    for (int k = 2; k <= npow2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int t = t0; t < (npow2 >> 1); t += nt) {
                const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
                const int l = i | j;
                const bool up = (i & k) == 0;
                const uint64_t a = sk[i], b = sk[l];
                if ((a > b) == up) { sk[i] = b; sk[l] = a; }
            }
            Sync::wait();
        }
    }
}

struct WarpSync {
    static __device__ __forceinline__ void wait() { __syncwarp(); }
};
struct CtaSync {
    static __device__ __forceinline__ void wait() { __syncthreads(); }
};

// One warp sorts npow2 (a power of two) keys in shared memory ascending, __syncwarp between
// stages.  The caller syncs the warp before (keys written) and reads the result after.
__device__ __forceinline__ void bitonic_in_shared(uint64_t* sk, int npow2, int lane) {
    bitonic_network_shared<WarpSync>(sk, npow2, lane, 32);
}

// The same network over the whole CTA, __syncthreads between stages.  Every thread of the block
// calls it; the caller syncs the block before (keys written) and reads the result after.
__device__ __forceinline__ void bitonic_in_cta(uint64_t* sk, int npow2) {
    bitonic_network_shared<CtaSync>(sk, npow2, int(threadIdx.x), int(blockDim.x));
}

// Rows of up to 512 keys: the same network with the keys in REGISTERS.  Lane L holds the KPL
// consecutive elements L*KPL .. L*KPL + KPL-1, so compare-exchange distances j < KPL stay inside
// a thread and j >= KPL are one shuffle per key with lane L ^ (j / KPL): no shared memory, no
// bank conflicts, no __syncwarp between stages (the shared-memory network above spends its time
// there).  Every lane of the warp must call it.
__device__ __forceinline__ uint64_t shfl_xor_u64(uint64_t v, int m) {
    uint32_t lo = uint32_t(v), hi = uint32_t(v >> 32);
    asm volatile("shfl.sync.bfly.b32 %0, %0, %2, 0x1f, 0xffffffff;\n\t"
                 "shfl.sync.bfly.b32 %1, %1, %2, 0x1f, 0xffffffff;"
                 : "+r"(lo), "+r"(hi) : "r"(m));
    return (uint64_t(hi) << 32) | lo;
}

__device__ __forceinline__ uint64_t shfl_u64(uint64_t v, int src) {
    const uint32_t lo = __shfl_sync(0xffffffffu, uint32_t(v), src);
    const uint32_t hi = __shfl_sync(0xffffffffu, uint32_t(v >> 32), src);
    return (uint64_t(hi) << 32) | lo;
}

template <int KPL>
__device__ __forceinline__ void bitonic_in_registers(uint64_t (&key)[KPL], int lane) {
    constexpr int N = KPL * 32;
#pragma unroll
    for (int k = 2; k <= N; k <<= 1) {
        // sort direction of the k-block the element sits in: bit k of i = L*KPL + r
        const bool lane_up = (k >= N) ? true : ((lane & (k >= KPL ? k / KPL : 1)) == 0);
#pragma unroll
        for (int j = k >> 1; j > 0; j >>= 1) {
            if (j >= KPL) {
                const int m = j / KPL;
                const bool keep_min = ((lane & m) == 0) == lane_up;
#pragma unroll
                for (int r = 0; r < KPL; ++r) {
                    const uint64_t o = shfl_xor_u64(key[r], m);
                    key[r] = ((o < key[r]) == keep_min) ? o : key[r];
                }
            } else {
#pragma unroll
                for (int r = 0; r < KPL; ++r) {
                    if ((r & j) == 0) {
                        const bool up = (k < KPL) ? ((r & k) == 0) : lane_up;
                        const uint64_t a = key[r], b = key[r | j];
                        const bool sw = (a > b) == up;
                        key[r] = sw ? b : a;
                        key[r | j] = sw ? a : b;
                    }
                }
            }
        }
    }
}

// sorted key i of a register-resident series after bitonic_in_registers (all lanes call it; i is
// warp-uniform)
template <int KPL>
__device__ __forceinline__ uint64_t pick_reg(const uint64_t (&key)[KPL], int i) {
    const int r = i % KPL;
    uint64_t v = key[0];
#pragma unroll
    for (int s = 1; s < KPL; ++s)
        if (r == s) v = key[s];
    return __shfl_sync(0xffffffffu, v, i / KPL);
}

// sorted key i of a register-resident series, where i may differ between lanes: KPL shuffles
template <int KPL>
__device__ __forceinline__ uint64_t pick_reg_lane(const uint64_t (&key)[KPL], int i) {
    uint64_t v = 0;
#pragma unroll
    for (int s = 0; s < KPL; ++s) {
        const uint64_t o = shfl_u64(key[s], i / KPL);
        if (i % KPL == s) v = o;
    }
    return v;
}

}  // namespace elfi
