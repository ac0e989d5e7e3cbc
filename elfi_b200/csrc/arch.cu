// arch.cu -- the ARCH(1) model of elfi/examples/arch.py in throughput mode: the simulator with its
// summaries fused, and the summaries of any (B, n) data.  arch.cuh has the arithmetic.
//
// Random streams (Philox4x32-10 keyed by the seed; counter (row, row >> 32, m, SALT_ARCH)),
// row = offset + i: block m gives the standard normals z_{2m}, z_{2m+1} (boxmuller.cuh, n0 then
// n1), where z_0 = e_0 and z_k = xi_k for 1 <= k <= n_obs; blocks 0 .. n_obs / 2 are drawn.  So
// every normal is a pure function of (seed, offset + row, k), whatever the batch split.  (The
// reference also draws xi_0, which it never uses; there is no such draw here.)
//
// Layout: one thread per row.  The row's n <= 128 observations are the state the three dependent
// reductions share (mean, then the variance about it, then the lagged products of the standardised
// values), so a thread keeps them in an observation-major shared-memory strip,
// strip[j * ARCH_THREADS + thread] (a warp's accesses hit 32 consecutive doubles: no bank
// conflicts).  The recurrence writes the strip once; arch_summaries then sweeps it 2 + L times and
// overwrites it with the standardised values.  The alternative, regenerating the row from its
// stream on each sweep, costs n Box-Muller pairs and square roots per sweep instead of one shared
// load.  The strip takes n KiB per block of 128 threads (100 KiB at the default n = 100).
//
// arch_summaries_kernel stages any strided row into the same strip and calls the same code, so the
// fused and the unfused summaries are the same bits by construction.
#include "arch.cuh"
#include "boxmuller.cuh"
#include "common.cuh"
#include "philox.cuh"

namespace elfi {

constexpr uint32_t SALT_ARCH = 0x41524348u;   // "ARCH"
constexpr int ARCH_THREADS = 128;

struct StripRow {
    double* p;
    ELFI_HD double& operator()(int j) const { return p[j * ARCH_THREADS]; }
};

// P[i * ldP + 0..1] = (t1, t2).  Y and S may be NULL.
__global__ void __launch_bounds__(ARCH_THREADS)
sim_arch_kernel(const double* __restrict__ P, int64_t ldP, int64_t B, int n_obs, int n_lags,
                uint64_t seed, uint64_t offset, double* __restrict__ Y, int64_t ldY,
                double* __restrict__ S, int64_t ldS) {
    extern __shared__ double strip_all[];
    const int64_t i = int64_t(blockIdx.x) * ARCH_THREADS + threadIdx.x;
    if (i >= B) return;
    const StripRow x{strip_all + threadIdx.x};
    const double t1 = P[i * ldP], t2 = P[i * ldP + 1];
    const Philox ph(seed);
    const uint64_t row = offset + uint64_t(i);
    const uint32_t r0 = uint32_t(row), r1 = uint32_t(row >> 32);
    double* y_out = Y ? Y + i * ldY : nullptr;
    double e = 0.0, y = 0.0;
    auto step = [&](int k, double xi) {   // observation k = 1 .. n_obs
        e = arch_e(xi, e, t2);
        y = arch_y(t1, y, e);
        if (S) x(k - 1) = y;
        if (y_out) y_out[k - 1] = y;
    };
    for (int m = 0; 2 * m <= n_obs; ++m) {
        double z0, z1;
        normal2(ph(r0, r1, uint32_t(m), SALT_ARCH), z0, z1);
        if (m == 0)
            e = z0;
        else
            step(2 * m, z0);
        if (2 * m + 1 <= n_obs) step(2 * m + 1, z1);
    }
    if (S) arch_summaries(n_obs, n_lags, x, S + i * ldS, 1);
}

// S[b * ldS + k] = summary k of the row X[b * ld_b + j * ld_j], j < n
__global__ void __launch_bounds__(ARCH_THREADS)
arch_summaries_kernel(const double* __restrict__ X, int64_t ld_b, int64_t ld_j, int64_t B, int n,
                      int n_lags, double* __restrict__ S, int64_t ldS) {
    extern __shared__ double strip_all[];
    const int64_t b = int64_t(blockIdx.x) * ARCH_THREADS + threadIdx.x;
    if (b >= B) return;
    const StripRow x{strip_all + threadIdx.x};
    const double* row = X + b * ld_b;
    for (int j = 0; j < n; ++j) x(j) = row[j * ld_j];
    arch_summaries(n, n_lags, x, S + b * ldS, 1);
}

static size_t arch_strip_bytes(int n) { return size_t(ARCH_THREADS) * n * sizeof(double); }

}  // namespace elfi

extern "C" {

int elfi_b200_sim_arch_f64(elfi_b200_ctx* ctx, const double* P, int64_t ldP, int64_t B,
                           int64_t n_obs, int64_t n_lags, uint64_t seed, uint64_t offset,
                           double* Y, int64_t ldY, double* S, int64_t ldS, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || P), "sim_arch: NULL argument");
    ELFI_REQUIRE(B >= 0 && ldP >= 2 && n_obs >= ARCH_NOBS_MIN && n_obs <= ARCH_NOBS_MAX &&
                     n_lags >= 1 && n_lags <= ARCH_LAGS_MAX && n_lags < n_obs,
                 "sim_arch: bad shape (%d <= n_obs <= %d, 1 <= n_lags <= min(%d, n_obs - 1), "
                 "ldP >= 2; B=%lld n_obs=%lld n_lags=%lld ldP=%lld)", ARCH_NOBS_MIN,
                 ARCH_NOBS_MAX, ARCH_LAGS_MAX, (long long)B, (long long)n_obs, (long long)n_lags,
                 (long long)ldP);
    ELFI_REQUIRE((Y == nullptr || ldY >= n_obs) && (S == nullptr || ldS >= arch_nsumm(int(n_lags))),
                 "sim_arch: bad leading dimension of Y or S");
    if (B == 0) return ELFI_B200_OK;
    const size_t smem = S ? arch_strip_bytes(int(n_obs)) : 0;
    const unsigned blocks = unsigned((B + ARCH_THREADS - 1) / ARCH_THREADS);
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        ELFI_CUDA_OK(cudaFuncSetAttribute(sim_arch_kernel,
                                          cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          int(arch_strip_bytes(ARCH_NOBS_MAX))));
        sim_arch_kernel<<<blocks, ARCH_THREADS, smem, stream>>>(P, ldP, B, int(n_obs), int(n_lags),
                                                                seed, offset, Y, ldY, S, ldS);
        return ELFI_B200_OK;
    });
}

int elfi_b200_arch_summaries_f64(elfi_b200_ctx* ctx, const double* X, int64_t ld_b, int64_t ld_j,
                                 int64_t B, int64_t n, int64_t n_lags, double* S, int64_t ldS,
                                 void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || (X && S)), "arch_summaries: NULL argument");
    ELFI_REQUIRE(B >= 0 && n >= ARCH_NOBS_MIN && n <= ARCH_NOBS_MAX && n_lags >= 1 &&
                     n_lags <= ARCH_LAGS_MAX && n_lags < n && ldS >= arch_nsumm(int(n_lags)),
                 "arch_summaries: bad shape (%d <= n <= %d, 1 <= n_lags <= min(%d, n - 1), "
                 "ldS >= 2 + L + L(L-1)/2; n=%lld n_lags=%lld ldS=%lld)", ARCH_NOBS_MIN,
                 ARCH_NOBS_MAX, ARCH_LAGS_MAX, (long long)n, (long long)n_lags, (long long)ldS);
    if (B == 0) return ELFI_B200_OK;
    const unsigned blocks = unsigned((B + ARCH_THREADS - 1) / ARCH_THREADS);
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        ELFI_CUDA_OK(cudaFuncSetAttribute(arch_summaries_kernel,
                                          cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          int(arch_strip_bytes(ARCH_NOBS_MAX))));
        arch_summaries_kernel<<<blocks, ARCH_THREADS, arch_strip_bytes(int(n)), stream>>>(
            X, ld_b, ld_j, B, int(n), int(n_lags), S, ldS);
        return ELFI_B200_OK;
    });
}

}  // extern "C"
