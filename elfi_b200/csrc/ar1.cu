// ar1.cu -- the AR(1) model of elfi/examples/ar1.py in throughput mode: the simulator, with the
// Euclidean distance of each series to the observed one fused into it.  ar1.cuh has the arithmetic.
//
// Random streams (Philox4x32-10 keyed by the seed; counter (row, row >> 32, m, SALT_AR1)),
// row = offset + i: block m gives the standard normals z_{2m}, z_{2m+1} (boxmuller.cuh, n0 then
// n1), and z_k is the innovation w_{k+1} of step k + 1, k < n_obs.  So every innovation is a pure
// function of (seed, offset + row, k), whatever the batch split.  (The reference also draws w_0,
// which it never uses; there is no such draw here.)
//
// Layout: one thread per row, the series in a register.  The reference's discrepancy reads the
// raw series, so the distance to the observed row y is accumulated as the series is generated,
// y_t read through the read-only cache (one address per warp and step: a broadcast).  With the
// distance fused a row costs its n_obs / 2 Philox blocks and writes 8 bytes (+ one mask bit)
// instead of 8 n_obs bytes written and read back.  When the series is asked for, each thread
// stores its row directly; the stores of a warp touch 32 rows, and L2 merges the partial sectors
// before they reach memory.  The acceptance epilogue is dist_record (distrecord.cuh) and the mask
// is compacted by launch_compact_mask, exactly as for ops.dist_euclid.
#include "ar1.cuh"
#include "boxmuller.cuh"
#include "distrecord.cuh"
#include "philox.cuh"

namespace elfi {

constexpr uint32_t SALT_AR1 = 0x41523120u;   // "AR1 "
constexpr int AR1_THREADS = 128;
constexpr int64_t AR1_NOBS_MAX = ELFI_B200_AR1_NOBS_MAX;
constexpr int64_t AR1_BATCH_MAX = ELFI_B200_AR1_BATCH_MAX;

// Row i: parameter phi[i], series X[i * ldX + t] (X may be NULL), distance to p.obs (p.obs may be
// NULL: then no distance and no mask).  Threads of rows >= B run to the epilogue: its ballot needs
// the whole warp.
__global__ void __launch_bounds__(AR1_THREADS)
sim_ar1_kernel(const double* __restrict__ phi_in, int64_t B, int n_obs, uint64_t seed,
               uint64_t offset, double* __restrict__ X, int64_t ldX, DistParams p) {
    const int64_t i = int64_t(blockIdx.x) * AR1_THREADS + threadIdx.x;
    double acc = 0.0;
    if (i < B) {
        const double phi = phi_in[i];
        const Philox ph(seed);
        const uint64_t row = offset + uint64_t(i);
        const uint32_t r0 = uint32_t(row), r1 = uint32_t(row >> 32);
        double* x_out = X ? X + i * ldX : nullptr;
        const double* __restrict__ y = p.obs;
        double x = 0.0;
        auto step = [&](int t, double w) {   // observation t = 0 .. n_obs - 1 (x_{t+1})
            x = ar1_step(phi, x, w);
            if (x_out) x_out[t] = x;
            if (y) acc = ar1_dist_term(acc, x, __ldg(y + t));
        };
        for (int m = 0; 2 * m < n_obs; ++m) {
            double z0, z1;
            normal2(ph(r0, r1, uint32_t(m), SALT_AR1), z0, z1);
            step(2 * m, z0);
            if (2 * m + 1 < n_obs) step(2 * m + 1, z1);
        }
    }
    if (p.obs != nullptr)
        dist_record<false, 1>(p, 1, i, B, threadIdx.x & 31,
                              [&](int) { return ar1_dist_finish(acc); });
}

}  // namespace elfi

extern "C" {

int elfi_b200_sim_ar1_f64(elfi_b200_ctx* ctx, const double* phi, int64_t B, int64_t n_obs,
                          uint64_t seed, uint64_t offset, double* X, int64_t ldX,
                          const double* obs, const double* thr_host, const double* thr_dev,
                          double* d_out, int32_t* acc_idx, int64_t* n_acc, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || phi), "sim_ar1: NULL argument");
    ELFI_REQUIRE(B >= 0 && B <= AR1_BATCH_MAX && n_obs >= 1 && n_obs <= AR1_NOBS_MAX,
                 "sim_ar1: bad shape (0 <= B <= %lld, 1 <= n_obs <= %lld; B=%lld n_obs=%lld)",
                 (long long)AR1_BATCH_MAX, (long long)AR1_NOBS_MAX, (long long)B,
                 (long long)n_obs);
    ELFI_REQUIRE(X == nullptr || ldX >= n_obs, "sim_ar1: ldX (%lld) < n_obs (%lld)",
                 (long long)ldX, (long long)n_obs);
    const bool thr = thr_host != nullptr || thr_dev != nullptr;
    ELFI_REQUIRE(thr_host == nullptr || thr_dev == nullptr,
                 "sim_ar1: thresholds on the host and on the device");
    ELFI_REQUIRE(obs != nullptr || (!thr && d_out == nullptr),
                 "sim_ar1: a distance or thresholds need the observed row");
    ELFI_REQUIRE(obs == nullptr || B == 0 || d_out != nullptr, "sim_ar1: d_out is NULL");
    ELFI_REQUIRE((acc_idx == nullptr && n_acc == nullptr) || thr,
                 "sim_ar1: acc_idx and n_acc require thresholds");
    if (B == 0) {
        if (n_acc) {
            return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
                return launch_compact_mask(nullptr, 0, acc_idx, n_acc, stream);
            });
        }
        return ELFI_B200_OK;
    }
    uint32_t* mask = nullptr;
    if (thr) {
        ELFI_CUDA_OK(cudaSetDevice(ctx->device));
        mask = static_cast<uint32_t*>(ctx_scratch(ctx, size_t((B + 31) / 32) * 4 + 256));
        if (!mask) return ELFI_B200_ERR_NOMEM;
    }
    const DistParams p = dist_params(obs, nullptr, 1, thr_host, thr_dev, d_out, mask);
    const unsigned blocks = unsigned((B + AR1_THREADS - 1) / AR1_THREADS);
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        sim_ar1_kernel<<<blocks, AR1_THREADS, 0, stream>>>(phi, B, int(n_obs), seed, offset, X,
                                                           ldX, p);
        ELFI_CUDA_OK(cudaGetLastError());
        if (thr && (acc_idx != nullptr || n_acc != nullptr))
            return launch_compact_mask(mask, B, acc_idx, n_acc, stream);
        return ELFI_B200_OK;
    });
}

}  // extern "C"
