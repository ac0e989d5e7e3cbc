// svm.cu -- the alpha-stable stochastic volatility model of
// elfi/examples/stochastic_volatility_model.py in throughput mode: the simulator with its quantile
// kurtosis and skewness fused.  svm.cuh and stable.cuh have the arithmetic.
//
// Random streams (Philox4x32-10 keyed by the seed), row = offset + i:
//   counter (row, row >> 32, j, SALT_SVM)     observation j's shock: TH = (1 - u01(x, y)) * pi - pi/2
//                                             (uniform on [-pi/2, pi/2)) and W = -log(u01(z, w));
//   counter (row, row >> 32, m, SALT_SVM_N)   the log-volatility normals z_{2m}, z_{2m+1}
//                                             (boxmuller.cuh, n0 then n1); z_t drives x_t.
// So every draw is a pure function of (seed, offset + row, j), whatever the batch split.  (The
// reference draws all normals of the batch t-major, then all angles, then all exponentials.)
//
// Layout: mg1.cu's.  x_t is sequential in t, so one thread simulates one row; the quantiles need
// the whole row sorted, which one warp does in registers.  Thread r writes its row to a per-warp
// shared-memory strip, strip[r * npad + j] (npad = n | 1: no bank conflicts; rowquantiles.cuh's
// warp_strips, here with at most SVM_WARPS_MAX warps in SVM_STRIP_BUDGET bytes per block); the
// warp then loads each row in turn, lane L taking elements k * 32 + L, sorts it (rowquantiles.cuh),
// lanes 0..4 pick the levels 0.05, 0.25, 0.5, 0.75, 0.95 and lane 0 writes S[b, 0:2] = (kurt,
// skew).  The data reaches HBM only when asked for, copied out of the strip row by row (coalesced).
// The fused summaries are those of ops.svm_summaries (row_quantiles of the data, then the same
// IEEE arithmetic) bit for bit, as a sorted row does not depend on the order its keys came in.
#include "boxmuller.cuh"
#include "common.cuh"
#include "philox.cuh"
#include "rowquantiles.cuh"
#include "svm.cuh"

namespace elfi {

constexpr uint32_t SALT_SVM = 0x53564d31u;     // "SVM1"
constexpr uint32_t SALT_SVM_N = 0x53564d4eu;   // "SVMN"
constexpr int SVM_WARPS_MAX = 4;
constexpr size_t SVM_STRIP_BUDGET = 64 * 1024;

// P[i * ldP + 0..6] = (alpha, beta, kappa, eta, mu, phi, sigma).  Y and S may be NULL.
// blockDim.x = 32 * warps.
template <int KPL>
__global__ void __launch_bounds__(32 * SVM_WARPS_MAX)
sim_svm_kernel(const double* __restrict__ P, int64_t ldP, int64_t B, int n, int npad,
               uint64_t seed, uint64_t offset, double* __restrict__ Y, int64_t ldY,
               double* __restrict__ S, int64_t ldS) {
    extern __shared__ double strip_all[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double* strip = strip_all + size_t(warp) * 32 * npad;
    const int64_t row0 = (int64_t(blockIdx.x) * (blockDim.x >> 5) + warp) * 32;
    if (row0 >= B) return;                           // warp-uniform
    const int64_t i = row0 + lane;
    if (i < B) {
        const double* p = P + i * ldP;
        const double alpha = p[0], beta = p[1], kappa = p[2], eta = p[3];
        const double mu = p[4], phi = p[5], sigma = p[6];
        const double scale0 = svm_stationary_scale(phi, sigma);
        const bool ok = svm_params_ok(alpha, beta, kappa, sigma, scale0);
        const StableRow sr = stable_row(alpha, beta, eta, kappa, true);
        const Philox ph(seed);
        const uint64_t row = offset + uint64_t(i);
        const uint32_t r0 = uint32_t(row), r1 = uint32_t(row >> 32);
        double* mine = strip + lane * npad;
        double x = 0.0;
        for (int m = 0; 2 * m < n; ++m) {
            double z[2];
            normal2(ph(r0, r1, uint32_t(m), SALT_SVM_N), z[0], z[1]);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int j = 2 * m + h;
                if (j < n) {
                    x = j == 0 ? svm_x0(z[0], mu, scale0) : svm_ar1(z[h], x, mu, phi, sigma);
                    const uint4 r = ph(r0, r1, uint32_t(j), SALT_SVM);
                    const double TH = stable_theta(1.0 - u01(r.x, r.y));
                    const double W = stable_expon(u01(r.z, r.w));
                    mine[j] = ok ? svm_y(x, stable_draw(sr, TH, W)) : NAN;
                }
            }
        }
    }
    __syncwarp();
    const int rows = int(B - row0 < 32 ? B - row0 : 32);
    if (Y)
        for (int r = 0; r < rows; ++r)
            for (int j = lane; j < n; j += 32) Y[(row0 + r) * ldY + j] = strip[r * npad + j];
    if (S) {
        const ToadPick pk = toad_quantile_pick(n, svm_level(lane < SVM_NQ ? lane : 0));
        for (int r = 0; r < rows; ++r) {
            uint64_t key[KPL];
#pragma unroll
            for (int k = 0; k < KPL; ++k) {
                const int j = k * 32 + lane;
                key[k] = j < n ? key_to_u64(strip[r * npad + j]) : ~uint64_t(0);
            }
            const double v = quantile_of_keys<KPL>(key, lane, n, pk);
            const double q05 = __shfl_sync(0xffffffffu, v, 0);
            const double q25 = __shfl_sync(0xffffffffu, v, 1);
            const double q50 = __shfl_sync(0xffffffffu, v, 2);
            const double q75 = __shfl_sync(0xffffffffu, v, 3);
            const double q95 = __shfl_sync(0xffffffffu, v, 4);
            double* s = S + (row0 + r) * ldS;
            if (lane == 0) s[0] = svm_kurt(q05, q25, q75, q95);
            if (lane == 1) s[1] = svm_skew(q05, q50, q95);
        }
    }
}

}  // namespace elfi

extern "C" {

int elfi_b200_sim_svm_f64(elfi_b200_ctx* ctx, const double* P, int64_t ldP, int64_t B,
                          int64_t n_obs, uint64_t seed, uint64_t offset, double* Y, int64_t ldY,
                          double* S, int64_t ldS, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || P), "sim_svm: NULL argument");
    ELFI_REQUIRE(B >= 0 && ldP >= SVM_NPARAMS && n_obs >= MG1_NOBS_MIN && n_obs <= MG1_NOBS_MAX &&
                     (S == nullptr || ldS >= SVM_NSUMM) && (Y == nullptr || ldY >= n_obs),
                 "sim_svm: bad shape (%d <= n_obs <= %d, ldP >= %d, ldS >= %d, ldY >= n_obs; "
                 "B=%lld n_obs=%lld ldP=%lld)", MG1_NOBS_MIN, MG1_NOBS_MAX, SVM_NPARAMS,
                 SVM_NSUMM, (long long)B, (long long)n_obs, (long long)ldP);
    if (B == 0 || (Y == nullptr && S == nullptr)) return ELFI_B200_OK;
    const int n = int(n_obs);
    const WarpStrips st = warp_strips(B, n, SVM_STRIP_BUDGET, SVM_WARPS_MAX);
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        return with_pow2<1, 16>(kpl_for(n, 1), [&](auto K) {
            ELFI_CUDA_OK(cudaFuncSetAttribute(sim_svm_kernel<decltype(K)::value>,
                                              cudaFuncAttributeMaxDynamicSharedMemorySize,
                                              int(st.smem)));
            sim_svm_kernel<decltype(K)::value><<<st.blocks, 32 * st.warps, st.smem, stream>>>(
                P, ldP, B, n, st.npad, seed, offset, Y, ldY, S, ldS);
            return ELFI_B200_OK;
        });
    });
}

}  // extern "C"
