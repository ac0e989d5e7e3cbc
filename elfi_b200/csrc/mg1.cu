// mg1.cu -- the M/G/1 queue of elfi/examples/mg1.py in throughput mode: the simulator with its
// quantile summaries fused, and the quantiles of the rows of any (B, n) matrix.  mg1.cuh has the
// arithmetic.
//
// Random streams (Philox4x32-10 keyed by the seed; counter (row, row >> 32, j, SALT_MG1)),
// row = offset + i: block j gives customer j's uniforms, u = u01(x, y) for the inter-arrival time
// and u' = u01(z, w) for the service time.  So every draw is a pure function of (seed, offset +
// row, j), whatever the batch split.  (The reference draws all inter-arrival times of the batch,
// then all service times.)
//
// Layout.  The recurrence is sequential in j, so one thread simulates one row; the quantiles need
// the whole row sorted, which one warp does in registers (bitonic_in_registers).  A warp's 32 rows
// therefore go through a per-warp shared-memory strip (rowquantiles.cuh's warp_strips, which
// svm.cu shares): thread r writes its row to strip[r * npad + j] (npad = n | 1, an odd stride: no
// bank conflicts), then the warp loads each row in turn, lane L taking elements k * 32 + L
// (conflict-free; the order of the keys before the sort does not matter), sorts it and lane k < nq
// writes quantile k.  The data reaches HBM only when asked for, copied out of the strip row by row
// (coalesced).  A strip takes 256 npad bytes per warp; a block has as many warps (at most
// MG1_WARPS_MAX = 4) as fit in MG1_STRIP_BUDGET = 64 KiB.  Not measured: keeping each row's sort
// in the simulating thread (a register or shared-memory sort of n keys per thread) instead of the
// warp.
//
// row_quantiles_kernel loads any strided row into the same registers and calls the same code
// (rowquantiles.cuh, which svm.cu shares).  A sorted row does not depend on the order its keys came
// in, so the fused and the unfused quantiles are the same bits by construction.
#include "common.cuh"
#include "mg1.cuh"
#include "philox.cuh"
#include "rowquantiles.cuh"

namespace elfi {

constexpr uint32_t SALT_MG1 = 0x4d473151u;   // "MG1Q"
constexpr int MG1_WARPS_MAX = 4;
constexpr size_t MG1_STRIP_BUDGET = 64 * 1024;

// P[i * ldP + 0..2] = (t1, t2, t3).  Y and S may be NULL.  blockDim.x = 32 * warps.
template <int KPL>
__global__ void __launch_bounds__(32 * MG1_WARPS_MAX)
sim_mg1_kernel(const double* __restrict__ P, int64_t ldP, int64_t B, int n, int npad, int nq,
               const QuantileLevels Q, uint64_t seed, uint64_t offset, double* __restrict__ Y,
               int64_t ldY, double* __restrict__ S, int64_t ldS) {
    extern __shared__ double strip_all[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double* strip = strip_all + size_t(warp) * 32 * npad;
    const int64_t row0 = (int64_t(blockIdx.x) * (blockDim.x >> 5) + warp) * 32;
    if (row0 >= B) return;                           // warp-uniform
    const int64_t i = row0 + lane;
    if (i < B) {
        const double t1 = P[i * ldP], t2 = P[i * ldP + 1], t3 = P[i * ldP + 2];
        const double inv_t3 = gnk_div(1.0, t3), range = leaf_sub(t2, t1);
        const bool ok = mg1_params_ok(inv_t3, range);
        const Philox ph(seed);
        const uint64_t row = offset + uint64_t(i);
        const uint32_t r0 = uint32_t(row), r1 = uint32_t(row >> 32);
        double sum_w = 0.0, sum_x = 0.0;
        double* mine = strip + lane * npad;
        for (int j = 0; j < n; ++j) {
            const uint4 r = ph(r0, r1, uint32_t(j), SALT_MG1);
            const double y = mg1_step(sum_w, sum_x, mg1_gap(inv_t3, u01(r.x, r.y)),
                                      mg1_service(t1, range, u01(r.z, r.w)));
            mine[j] = ok ? y : NAN;
        }
    }
    __syncwarp();
    const int rows = int(B - row0 < 32 ? B - row0 : 32);
    if (Y)
        for (int r = 0; r < rows; ++r)
            for (int j = lane; j < n; j += 32) Y[(row0 + r) * ldY + j] = strip[r * npad + j];
    if (S) {
        const ToadPick pk = lane_pick(n, nq, Q, lane);
        for (int r = 0; r < rows; ++r) {
            uint64_t key[KPL];
#pragma unroll
            for (int k = 0; k < KPL; ++k) {
                const int j = k * 32 + lane;
                key[k] = j < n ? key_to_u64(strip[r * npad + j]) : ~uint64_t(0);
            }
            quantiles_of_keys<KPL>(key, lane, n, nq, pk, true, S + (row0 + r) * ldS);
        }
    }
}

// S[b * ldS + k] = quantile k of the row X[b * ld_b + j * ld_j], j < n; one warp per row, the
// loop bounds block-uniform so that the shuffles sit in convergent code
template <int KPL>
__global__ void __launch_bounds__(256, KPL >= 8 ? 1 : 2)
row_quantiles_kernel(const double* __restrict__ X, int64_t ld_b, int64_t ld_j, int64_t B, int n,
                     int nq, const QuantileLevels Q, double* __restrict__ S, int64_t ldS) {
    const int lane = threadIdx.x & 31;
    const ToadPick pk = lane_pick(n, nq, Q, lane);
    for (int64_t base = int64_t(blockIdx.x) * 8; base < B; base += int64_t(gridDim.x) * 8) {
        const int64_t b = base + (threadIdx.x >> 5);
        const bool live = b < B;
        const double* x = X + (live ? b : 0) * ld_b;
        uint64_t key[KPL];
#pragma unroll
        for (int k = 0; k < KPL; ++k) {
            const int j = k * 32 + lane;
            key[k] = (live && j < n) ? key_to_u64(__ldg(x + int64_t(j) * ld_j)) : ~uint64_t(0);
        }
        quantiles_of_keys<KPL>(key, lane, n, nq, pk, live, S + (live ? b : 0) * ldS);
    }
}

}  // namespace elfi

extern "C" {

int elfi_b200_sim_mg1_f64(elfi_b200_ctx* ctx, const double* P, int64_t ldP, int64_t B,
                          int64_t n_obs, int64_t nq, const double* q_host, uint64_t seed,
                          uint64_t offset, double* Y, int64_t ldY, double* S, int64_t ldS,
                          void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || P) && (S == nullptr || q_host), "sim_mg1: NULL argument");
    ELFI_REQUIRE(B >= 0 && ldP >= 3 && n_obs >= MG1_NOBS_MIN && n_obs <= MG1_NOBS_MAX &&
                     (S == nullptr || (nq >= 1 && nq <= MG1_NQ_MAX && ldS >= nq)) &&
                     (Y == nullptr || ldY >= n_obs),
                 "sim_mg1: bad shape (%d <= n_obs <= %d, 1 <= nq <= %d, ldP >= 3, ldS >= nq, "
                 "ldY >= n_obs; n_obs=%lld nq=%lld ldP=%lld)", MG1_NOBS_MIN, MG1_NOBS_MAX,
                 MG1_NQ_MAX, (long long)n_obs, (long long)nq, (long long)ldP);
    QuantileLevels Q;
    ELFI_REQUIRE(S == nullptr || quantile_levels(q_host, nq, &Q),
                 "sim_mg1: every q must lie in [0, 1]");
    if (S == nullptr) memset(&Q, 0, sizeof(Q));
    if (B == 0) return ELFI_B200_OK;
    const int n = int(n_obs);
    const WarpStrips st = warp_strips(B, n, MG1_STRIP_BUDGET, MG1_WARPS_MAX);
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        return with_pow2<1, 16>(kpl_for(n, 1), [&](auto K) {
            ELFI_CUDA_OK(cudaFuncSetAttribute(sim_mg1_kernel<decltype(K)::value>,
                                              cudaFuncAttributeMaxDynamicSharedMemorySize,
                                              int(st.smem)));
            sim_mg1_kernel<decltype(K)::value><<<st.blocks, 32 * st.warps, st.smem, stream>>>(
                P, ldP, B, n, st.npad, int(nq), Q, seed, offset, Y, ldY, S, ldS);
            return ELFI_B200_OK;
        });
    });
}

int elfi_b200_row_quantiles_f64(elfi_b200_ctx* ctx, const double* X, int64_t ld_b, int64_t ld_j,
                                int64_t B, int64_t n, int64_t nq, const double* q_host, double* S,
                                int64_t ldS, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && q_host && (B == 0 || (X && S)), "row_quantiles: NULL argument");
    ELFI_REQUIRE(B >= 0 && n >= MG1_NOBS_MIN && n <= MG1_NOBS_MAX && nq >= 1 && nq <= MG1_NQ_MAX &&
                     ldS >= nq,
                 "row_quantiles: bad shape (%d <= n <= %d, 1 <= nq <= %d, ldS >= nq; n=%lld "
                 "nq=%lld ldS=%lld)", MG1_NOBS_MIN, MG1_NOBS_MAX, MG1_NQ_MAX, (long long)n,
                 (long long)nq, (long long)ldS);
    QuantileLevels Q;
    ELFI_REQUIRE(quantile_levels(q_host, nq, &Q), "row_quantiles: every q must lie in [0, 1]");
    if (B == 0) return ELFI_B200_OK;
    const int64_t want = (B + 7) / 8;
    const unsigned blocks = unsigned(want < 65535 * 16 ? want : 65535 * 16);
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        with_pow2<1, 16>(kpl_for(int(n), 1), [&](auto K) {
            row_quantiles_kernel<decltype(K)::value><<<blocks, 256, 0, stream>>>(
                X, ld_b, ld_j, B, int(n), int(nq), Q, S, ldS);
        });
        return ELFI_B200_OK;
    });
}

}  // extern "C"
