// distrecord.cuh -- what every kernel that ends in a distance and an acceptance test shares: the
// kernel parameters (DistParams, dist_params), the acceptance epilogue (dist_record) and the
// compaction of its mask into ascending row indices (launch_compact_mask, in distance.cu).  The
// distance kernels (distance.cu) and the simulators with a fused distance (ar1.cu) use them, so a
// fused distance is accepted and compacted exactly as ops.dist_euclid does it.
#pragma once

#include "common.cuh"

namespace elfi {

struct DistParams {
    const double* obs;   // (D)
    const double* W;     // (K, D) or nullptr
    double* d_out;       // (B, K)
    uint32_t* mask;      // ceil(B/32) words or nullptr
    int K;
    int has_thr;
    const double* shift_src;   // fused column moments: row 0 of S (the shift of the power sums)
    double* mom_partial;       // (warps, 2, D) shifted power sums per warp, or nullptr
    const double* thr_dev;   // K thresholds in device memory (e.g. a quantile computed on the
                             // device), or nullptr: then thr[] below, copied from the host
    double thr[ELFI_B200_MAX_NESTED];
    __device__ __forceinline__ double threshold(int k) const {
        return thr_dev ? __ldg(thr_dev + k) : thr[k];
    }
};

// The acceptance epilogue of every distance kernel: store the row's K distances, compare each
// with its threshold, ballot, lane 0 writes the warp's mask word.  `column(k)` turns the caller's
// accumulator k into the finished distance; it runs for rows < B only.
// KMAX is a compile-time bound so that the caller's acc[] and thr[] are indexed by constants (a
// runtime-indexed acc[] would be demoted to local memory); with KMAX = 0 the loop runs to K
// instead, for a caller that computes a whole column inside `column`.
// WHOLE_WARP: row-stream consumers run full warps over zero-filled tiles and always own their
// mask word; a thread-per-row grid may end in a warp that starts at or beyond B and owns none.
template <bool WHOLE_WARP, int KMAX, class Column>
__device__ __forceinline__ void dist_record(const DistParams& p, int K, int64_t row, int64_t B,
                                            int lane, Column column) {
    bool ok = row < B;
    if (ok) {
#pragma unroll
        for (int k = 0; k < (KMAX ? KMAX : K); ++k) {
            if (k < K) {
                const double d = column(k);
                p.d_out[row * K + k] = d;
                if (p.has_thr) ok = ok && (d <= p.threshold(k));
            }
        }
    }
    if (p.mask != nullptr) {
        const uint32_t bits = __ballot_sync(0xffffffffu, ok && p.has_thr);
        if (lane == 0 && (WHOLE_WARP || (row - lane) < B)) p.mask[row >> 5] = bits;
    }
}

// The kernel parameters of one call.  Thresholds come from the host (copied into thr[]), stay on
// the device, or there are none.
inline DistParams dist_params(const double* obs, const double* W, int64_t K,
                              const double* thr_host, const double* thr_dev, double* d_out,
                              uint32_t* mask) {
    DistParams p = {};
    p.obs = obs;
    p.W = W;
    p.d_out = d_out;
    p.mask = mask;
    p.K = int(K);
    p.has_thr = thr_host != nullptr || thr_dev != nullptr;
    p.thr_dev = thr_dev;
    if (thr_host)
        for (int k = 0; k < K; ++k) p.thr[k] = thr_host[k];
    return p;
}

// Mask words of B rows -> ascending accepted row indices idx (may be NULL) and their number n_out
// (may be NULL), on `stream`.
int launch_compact_mask(const uint32_t* mask, int64_t B, int32_t* idx, int64_t* n_out,
                        cudaStream_t stream);

}  // namespace elfi
