// ricker.cu -- the Ricker population model of elfi/examples/ricker.py in throughput mode: Poisson
// draws (poisson.cuh), the deterministic and stochastic simulators with the summaries
// [np.mean, np.var, num_zeros] fused in, the zero count of a data matrix and the discrepancy
// chi_squared.
//
// Random streams (Philox4x32-10 keyed by the seed; counter (row, row >> 32, block, salt)):
//   poisson_kernel     element i: row = offset + i, block j = PTRS trial j (inversion uses block 0)
//   sim_ricker_kernel  row = offset + i; step t (0 <= t < n_obs) uses blocks (t << 8) | j:
//                        j = 0      e_t = first Box-Muller normal of the block (boxmuller.cuh)
//                        j = 1 + m  block m of the Poisson draw of Y_t (m < POISSON_MAX_TRIALS)
// so every value is a pure function of (seed, offset + row, t, trial), whatever the sharding.
//
// Stochastic model (ricker.py:43-85), N_{-1} = stock_init:
//   N_t = N_{t-1} * exp((r - N_{t-1}) + (sigma * e_t)),   Y_t ~ Poisson(phi * N_t)
// Deterministic model (ricker.py:11-40): Y_0 = stock_init, Y_t = Y_{t-1} * exp(r - Y_{t-1}).
// Each operation is rounded on its own, in the reference's order (no FMA contraction).
//
// Fused summaries (n_obs <= RICKER_FUSED_MAX = 128, one leaf of NumPy's pairwise sum): a thread
// keeps its row's Y in an observation-major shared-memory strip, strip[t * 128 + thread] (a warp's
// reads and writes hit 32 consecutive doubles: no bank conflicts), counts the zeros as it goes,
// then sums the strip twice in LeafSum order: mean = sum / n, var = sum((y - mean)^2) / n, the
// bits of ops.meanvar.  The strip takes 1 KiB per observation and block.
#include "boxmuller.cuh"
#include "common.cuh"
#include "leafsum.cuh"
#include "philox.cuh"
#include "poisson.cuh"

namespace elfi {

constexpr uint32_t SALT_POISSON = 0x504f4953u;   // "POIS"
constexpr uint32_t SALT_RICKER = 0x5249434bu;    // "RICK"
constexpr int RICKER_FUSED_MAX = ELFI_B200_RICKER_FUSED_MAX;
static_assert(RICKER_FUSED_MAX == LEAF_MAX_TERMS, "the fused summaries sum one pairwise leaf");
constexpr int RICKER_THREADS = 128;
// t << 8 fits the 32-bit block word
constexpr int64_t RICKER_NOBS_MAX = ELFI_B200_RICKER_NOBS_MAX;

__global__ void __launch_bounds__(256)
poisson_kernel(const double* __restrict__ lam, int64_t n, uint64_t seed, uint64_t offset,
               double* __restrict__ out) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Philox ph(seed);
    const uint64_t row = offset + uint64_t(i);
    const uint32_t r0 = uint32_t(row), r1 = uint32_t(row >> 32);
    out[i] = poisson_draw(lam[i], [&](int j) { return ph(r0, r1, uint32_t(j), SALT_POISSON); }).k;
}

// sum_j f(strip[j * RICKER_THREADS]) over a row of the strip, f = identity (mean) or the squared
// deviation from `mean`, in LeafSum order
template <int J>
__device__ __forceinline__ void push_strip(LeafSum& s, int j0, int n, const double* strip, bool sq,
                                           double mean) {
    const int j = j0 + J;
    if (j < n) {
        const double y = strip[j * RICKER_THREADS];
        const double c = __dsub_rn(y, mean);
        s.push<J>(j, sq ? __dmul_rn(c, c) : y);
    }
    if constexpr (J + 1 < 8) push_strip<J + 1>(s, j0, n, strip, sq, mean);
}

// One thread per row.  P[i * ldP + ...] = (r, sigma, phi) (STOCH) or (r).  Y, N, S may be NULL.
// Without the minimum of 4 blocks per SM ptxas caps the fused kernel at 64 registers and spills.
template <bool STOCH, bool SUMM>
__global__ void __launch_bounds__(RICKER_THREADS, 4)
sim_ricker_kernel(const double* __restrict__ P, int64_t ldP, int64_t B, int n_obs, double stock_init,
                  uint64_t seed, uint64_t offset, double* __restrict__ Y, int64_t ldY,
                  double* __restrict__ N, int64_t ldN, double* __restrict__ S, int64_t ldS) {
    extern __shared__ double strip_all[];
    const int64_t i = int64_t(blockIdx.x) * RICKER_THREADS + threadIdx.x;
    if (i >= B) return;
    double* strip = strip_all + threadIdx.x;
    const double r = P[i * ldP];
    const double sigma = STOCH ? P[i * ldP + 1] : 0.0;
    const double phi = STOCH ? P[i * ldP + 2] : 0.0;
    const Philox ph(seed);
    const uint64_t row = offset + uint64_t(i);
    const uint32_t r0 = uint32_t(row), r1 = uint32_t(row >> 32);
    double stock = stock_init;
    double zeros = 0.0;
    for (int t = 0; t < n_obs; ++t) {
        double y;
        if (STOCH) {
            const uint32_t base = uint32_t(t) << 8;
            double e, e1;
            normal2(ph(r0, r1, base, SALT_RICKER), e, e1);
            stock = __dmul_rn(stock, exp(__dadd_rn(__dsub_rn(r, stock), __dmul_rn(sigma, e))));
            y = poisson_draw(__dmul_rn(phi, stock), [&](int j) {
                    return ph(r0, r1, base | uint32_t(1 + j), SALT_RICKER);
                }).k;
        } else {
            if (t > 0) stock = __dmul_rn(stock, exp(__dsub_rn(r, stock)));
            y = stock;
        }
        if (Y) Y[i * ldY + t] = y;
        if (N) N[i * ldN + t] = stock;
        if (SUMM) {
            strip[t * RICKER_THREADS] = y;
            zeros += (y == 0.0) ? 1.0 : 0.0;
        }
    }
    if (SUMM) {
        LeafSum s;
        s.begin(n_obs);
        for (int j0 = 0; j0 < n_obs; j0 += 8) push_strip<0>(s, j0, n_obs, strip, false, 0.0);
        const double mean = s.finish(n_obs) / double(n_obs);
        s.begin(n_obs);
        for (int j0 = 0; j0 < n_obs; j0 += 8) push_strip<0>(s, j0, n_obs, strip, true, mean);
        S[i * ldS] = mean;
        S[i * ldS + 1] = s.finish(n_obs) / double(n_obs);
        S[i * ldS + 2] = zeros;
    }
}

// out[i * ld_out] = number of zeros in row i of X (B, n): one warp per row
__global__ void __launch_bounds__(256)
count_zeros_kernel(const double* __restrict__ X, int64_t ldX, int64_t B, int64_t n,
                   double* __restrict__ out, int64_t ld_out) {
    const int lane = threadIdx.x & 31;
    for (int64_t row = int64_t(blockIdx.x) * 8 + (threadIdx.x >> 5); row < B;
         row += int64_t(gridDim.x) * 8) {
        const double* x = X + row * ldX;
        unsigned c = 0;
        for (int64_t j = lane; j < n; j += 32) c += (x[j] == 0.0) ? 1u : 0u;
        c = __reduce_add_sync(0xffffffffu, c);
        if (lane == 0) out[row * ld_out] = double(c);
    }
}

// chi_squared: sum_j (S[i, j] - obs[j])^2 / obs[j] in NumPy's pairwise order
template <int J>
__device__ __forceinline__ void push_chi(LeafSum& s, int j0, int K, const double* row,
                                         const double* obs) {
    const int j = j0 + J;
    if (j < K) {
        const double t = __dsub_rn(row[j], obs[j]);
        s.push<J>(j, __ddiv_rn(__dmul_rn(t, t), obs[j]));
    }
    if constexpr (J + 1 < 8) push_chi<J + 1>(s, j0, K, row, obs);
}

__global__ void __launch_bounds__(256)
chi_squared_kernel(const double* __restrict__ S, int64_t ldS, int64_t B, int K,
                   const double* __restrict__ obs, double* __restrict__ out) {
    const int64_t stride = int64_t(gridDim.x) * blockDim.x;
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < B; i += stride) {
        LeafSum s;
        s.begin(K);
        for (int j0 = 0; j0 < K; j0 += 8) push_chi<0>(s, j0, K, S + i * ldS, obs);
        out[i] = s.finish(K);
    }
}

template <bool STOCH, bool SUMM>
static int launch_sim_ricker(const double* P, int64_t ldP, int64_t B, int n, double stock_init,
                             uint64_t seed, uint64_t offset, double* Y, int64_t ldY, double* N,
                             int64_t ldN, double* S, int64_t ldS, cudaStream_t stream) {
    const size_t smem = SUMM ? size_t(RICKER_THREADS) * n * sizeof(double) : 0;
    if (SUMM)
        ELFI_CUDA_OK(cudaFuncSetAttribute(sim_ricker_kernel<STOCH, SUMM>,
                                          cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    const unsigned blocks = unsigned((B + RICKER_THREADS - 1) / RICKER_THREADS);
    sim_ricker_kernel<STOCH, SUMM><<<blocks, RICKER_THREADS, smem, stream>>>(
        P, ldP, B, n, stock_init, seed, offset, Y, ldY, N, ldN, S, ldS);
    return ELFI_B200_OK;
}

}  // namespace elfi

extern "C" {

int elfi_b200_poisson_f64(elfi_b200_ctx* ctx, const double* lam, int64_t n, uint64_t seed,
                          uint64_t offset, double* out, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && n >= 0 && (n == 0 || (lam && out)), "poisson: bad argument");
    if (n == 0) return ELFI_B200_OK;
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        poisson_kernel<<<unsigned((n + 255) / 256), 256, 0, stream>>>(lam, n, seed, offset, out);
        return ELFI_B200_OK;
    });
}

int elfi_b200_sim_ricker_f64(elfi_b200_ctx* ctx, const double* P, int64_t ldP, int64_t n_params,
                             int64_t B, int64_t n_obs, double stock_init, uint64_t seed,
                             uint64_t offset, double* Y, int64_t ldY, double* N, int64_t ldN,
                             double* S, int64_t ldS, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || P), "sim_ricker: NULL argument");
    ELFI_REQUIRE(n_params == 1 || n_params == 3,
                 "sim_ricker: 3 parameters (stochastic) or 1 (deterministic), got %lld",
                 (long long)n_params);
    ELFI_REQUIRE(B >= 0 && n_obs >= 1 && n_obs <= RICKER_NOBS_MAX && ldP >= n_params,
                 "sim_ricker: bad shape (1 <= n_obs <= %lld; B=%lld n_obs=%lld ldP=%lld)",
                 (long long)RICKER_NOBS_MAX, (long long)B, (long long)n_obs, (long long)ldP);
    ELFI_REQUIRE((Y == nullptr || ldY >= n_obs) && (N == nullptr || ldN >= n_obs),
                 "sim_ricker: bad leading dimension of Y or N");
    ELFI_REQUIRE(S == nullptr || (n_obs <= RICKER_FUSED_MAX && ldS >= 3),
                 "sim_ricker: fused summaries need n_obs <= %d and ldS >= 3 (n_obs=%lld)",
                 RICKER_FUSED_MAX, (long long)n_obs);
    if (B == 0) return ELFI_B200_OK;
    const int n = int(n_obs);
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        if (n_params == 3)
            return S ? launch_sim_ricker<true, true>(P, ldP, B, n, stock_init, seed, offset, Y, ldY, N, ldN, S, ldS, stream)
                     : launch_sim_ricker<true, false>(P, ldP, B, n, stock_init, seed, offset, Y, ldY, N, ldN, S, ldS, stream);
        return S ? launch_sim_ricker<false, true>(P, ldP, B, n, stock_init, seed, offset, Y, ldY, N, ldN, S, ldS, stream)
                 : launch_sim_ricker<false, false>(P, ldP, B, n, stock_init, seed, offset, Y, ldY, N, ldN, S, ldS, stream);
    });
}

int elfi_b200_count_zeros_f64(elfi_b200_ctx* ctx, const double* X, int64_t ldX, int64_t B, int64_t n,
                              double* out, int64_t ld_out, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || (X && out)), "count_zeros: NULL argument");
    ELFI_REQUIRE(B >= 0 && n >= 1 && n < (int64_t(1) << 32) && ldX >= n && ld_out >= 1,
                 "count_zeros: bad shape (B=%lld n=%lld ldX=%lld)", (long long)B, (long long)n,
                 (long long)ldX);
    if (B == 0) return ELFI_B200_OK;
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        count_zeros_kernel<<<capped_grid(ctx, B, 8, 16), 256, 0, stream>>>(X, ldX, B, n, out,
                                                                           ld_out);
        return ELFI_B200_OK;
    });
}

int elfi_b200_chi_squared_f64(elfi_b200_ctx* ctx, const double* S, int64_t ldS, int64_t B, int64_t K,
                              const double* obs, double* out, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || (S && obs && out)), "chi_squared: NULL argument");
    ELFI_REQUIRE(B >= 0 && K >= 1 && K <= LEAF_MAX_TERMS && ldS >= K,
                 "chi_squared: bad shape (1 <= K <= %d; K=%lld)", LEAF_MAX_TERMS, (long long)K);
    if (B == 0) return ELFI_B200_OK;
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        chi_squared_kernel<<<capped_grid(ctx, B, 256, 16), 256, 0, stream>>>(S, ldS, B, int(K), obs,
                                                                             out);
        return ELFI_B200_OK;
    });
}

}  // extern "C"
