// sumsel.cu -- summary-statistic selection (TwoStageSelection, elfi/methods/diagnostics.py):
// the distance of every candidate combination from one read of each row, the k-th nearest
// neighbour radii and their log sum for many point sets, and the mean root sum of squared errors.
//
// Semantics and limits are stated in include/elfi_b200.h.  Every reduction has a fixed order and
// none uses atomics, so repeated calls give the same bits.
#include <cmath>

#include "metric.cuh"

namespace elfi {

// ---- all-combination distances ------------------------------------------------------------------
constexpr int SS_ROWS = 32;        // rows staged per CTA: one per lane
constexpr int SS_THREADS = 256;    // 8 warps take the combinations in turn
constexpr int SS_MAX_W = ELFI_B200_SUBSET_MAX_WIDTH;

// Rows are staged at an odd stride (W | 1 doubles), so the 32 lanes of a warp, each reading
// column j of its own row, hit different banks; obs[j] is one broadcast.
template <int METRIC>
__global__ void __launch_bounds__(SS_THREADS)
subset_distance_kernel(const double* __restrict__ S, int64_t ldS, int64_t B, int W,
                       const double* __restrict__ obs, const int32_t* __restrict__ ranges,
                       const int32_t* __restrict__ comb, int C, double* __restrict__ d_out,
                       int64_t ld_out) {
    extern __shared__ double ss_smem[];
    const int Wp = W | 1;
    double* rows = ss_smem;
    double* obs_s = ss_smem + SS_ROWS * Wp;
    for (int j = threadIdx.x; j < W; j += blockDim.x) obs_s[j] = obs[j];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
    const double* mine = rows + lane * Wp;
    for (int64_t r0 = int64_t(blockIdx.x) * SS_ROWS; r0 < B; r0 += int64_t(gridDim.x) * SS_ROWS) {
        const int nr = int(B - r0 < SS_ROWS ? B - r0 : SS_ROWS);
        __syncthreads();   // the previous tile is consumed
        for (int e = threadIdx.x; e < SS_ROWS * W; e += blockDim.x) {
            const int r = e / W, j = e - r * W;
            rows[r * Wp + j] = r < nr ? S[(r0 + r) * ldS + j] : 0.0;
        }
        __syncthreads();
        for (int c = warp; c < C; c += n_warps) {
            double acc = 0.0;
            const int g1 = __ldg(comb + c + 1);
            for (int g = __ldg(comb + c); g < g1; ++g) {
                const int col = __ldg(ranges + 2 * g), end = col + __ldg(ranges + 2 * g + 1);
                for (int j = col; j < end; ++j)
                    acc = metric_term<METRIC>(acc, __dsub_rn(mine[j], obs_s[j]), 0.0);
            }
            if (lane < nr) d_out[int64_t(c) * ld_out + r0 + lane] = metric_value<METRIC>(acc, 0.0);
        }
    }
}

template <int METRIC>
static int launch_subset_distance(elfi_b200_ctx* ctx, const double* S, int64_t ldS, int64_t B,
                                  int W, const double* obs, const int32_t* ranges,
                                  const int32_t* comb, int C, double* d_out, int64_t ld_out,
                                  cudaStream_t stream) {
    const size_t smem = (size_t(SS_ROWS) * (W | 1) + W) * sizeof(double);
    ELFI_CUDA_OK(cudaFuncSetAttribute(subset_distance_kernel<METRIC>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    const int fit = int(200 * 1024 / smem);    // CTAs whose staged rows fit one SM's shared memory
    const int per_sm = fit < 1 ? 1 : (fit > 8 ? 8 : fit);
    subset_distance_kernel<METRIC><<<capped_grid(ctx, B, SS_ROWS, per_sm), SS_THREADS, smem, stream>>>(
        S, ldS, B, W, obs, ranges, comb, C, d_out, ld_out);
    return ELFI_B200_OK;
}

// ---- k-th nearest neighbour radii ----------------------------------------------------------------
constexpr int KN_QUERIES = 128;    // query points (threads) per CTA
constexpr int KN_TILE = 256;       // set points per shared tile
constexpr int KN_MAX_Q = ELFI_B200_KNN_MAX_Q;
constexpr int KN_MAX_K = ELFI_B200_KNN_MAX_K;
constexpr int RED_THREADS = 256;

// best[] holds the KMAX smallest values seen, ascending.  Only the top k slots take part: the
// KMAX - k below them start at -inf and never move, so best[KMAX - 1] is the k-th smallest.
template <int KMAX>
__device__ __forceinline__ void insert_sorted(double (&best)[KMAX], double v) {
    if (!(v < best[KMAX - 1])) return;
#pragma unroll
    for (int s = KMAX - 1; s > 0; --s) best[s] = best[s - 1] > v ? best[s - 1] : fmin(best[s], v);
    best[0] = fmin(best[0], v);
}

template <int KMAX>
__global__ void __launch_bounds__(KN_QUERIES, 4)
knn_radius_kernel(const double* __restrict__ X, int64_t ldX, int n, int q, int k,
                  double* __restrict__ R) {
    __shared__ double tile[KN_TILE * KN_MAX_Q];
    const int64_t set = blockIdx.y;
    const double* Xs = X + set * n * ldX;
    const int i = blockIdx.x * KN_QUERIES + threadIdx.x;
    double x[KN_MAX_Q];
#pragma unroll
    for (int j = 0; j < KN_MAX_Q; ++j) x[j] = (i < n && j < q) ? Xs[int64_t(i) * ldX + j] : 0.0;
    double best[KMAX];
#pragma unroll
    for (int s = 0; s < KMAX; ++s) best[s] = s < KMAX - k ? -INFINITY : INFINITY;
    for (int t0 = 0; t0 < n; t0 += KN_TILE) {
        const int nt = n - t0 < KN_TILE ? n - t0 : KN_TILE;
        __syncthreads();
        for (int e = threadIdx.x; e < nt * q; e += blockDim.x) {
            const int p = e / q, j = e - p * q;
            tile[e] = Xs[int64_t(t0 + p) * ldX + j];
        }
        __syncthreads();
        for (int p = 0; p < nt; ++p) {
            const double* y = tile + p * q;
            double d2 = 0.0;
#pragma unroll
            for (int j = 0; j < KN_MAX_Q; ++j) {
                if (j < q) {
                    const double d = __dsub_rn(x[j], y[j]);
                    d2 = __dadd_rn(d2, __dmul_rn(d, d));
                }
            }
            insert_sorted<KMAX>(best, d2);
        }
    }
    if (i < n) R[set * n + i] = sqrt(best[KMAX - 1]);
}

// Sum of v over a CTA of RED_THREADS threads in a fixed pairwise order; the result is in red[0].
__device__ __forceinline__ void block_sum(double v, double* red) {
    red[threadIdx.x] = v;
#pragma unroll
    for (int h = RED_THREADS / 2; h > 0; h >>= 1) {
        __syncthreads();
        if (threadIdx.x < h) red[threadIdx.x] = __dadd_rn(red[threadIdx.x], red[threadIdx.x + h]);
    }
    __syncthreads();
}

__global__ void __launch_bounds__(RED_THREADS)
log_sum_kernel(const double* __restrict__ R, int n, double* __restrict__ logsum) {
    __shared__ double red[RED_THREADS];
    const double* Rs = R + int64_t(blockIdx.x) * n;
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += RED_THREADS) s = __dadd_rn(s, log(Rs[i]));
    block_sum(s, red);
    if (threadIdx.x == 0) logsum[blockIdx.x] = red[0];
}

// ---- mean root sum of squared errors -------------------------------------------------------------
__global__ void __launch_bounds__(RED_THREADS)
mrsse_kernel(const double* __restrict__ T, int64_t ldT, int64_t n, int q,
             const double* __restrict__ P, int64_t ldP, int64_t m, double* __restrict__ out) {
    __shared__ double red[RED_THREADS];
    const double* Ts = T + int64_t(blockIdx.x) * n * ldT;
    const int64_t nq = n * q;
    double total = 0.0;
    for (int64_t j = 0; j < m; ++j) {
        const double* pj = P + j * ldP;
        double s = 0.0;
        for (int64_t e = threadIdx.x; e < nq; e += RED_THREADS) {
            const int64_t i = e / q;
            const int l = int(e - i * q);
            const double d = __dsub_rn(Ts[i * ldT + l], pj[l]);
            s = __dadd_rn(s, __dmul_rn(d, d));
        }
        block_sum(s, red);
        if (threadIdx.x == 0) total = __dadd_rn(total, sqrt(red[0]));
    }
    if (threadIdx.x == 0) out[blockIdx.x] = __ddiv_rn(total, double(m));
}

}  // namespace elfi

extern "C" {

int elfi_b200_subset_distance_f64(elfi_b200_ctx* ctx, int32_t metric, const double* S, int64_t ldS,
                                  int64_t B, int64_t W, const double* obs, const int32_t* ranges,
                                  const int32_t* comb, int64_t C, double* d_out, int64_t ld_out,
                                  void* stream) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && obs && ranges && comb && d_out && (B == 0 || S),
                 "subset_distance: NULL argument");
    ELFI_REQUIRE(W >= 1 && W <= SS_MAX_W && ldS >= W && B >= 0 && B < (int64_t(1) << 31) &&
                     C >= 1 && C <= ELFI_B200_SUBSET_MAX_COMBINATIONS && ld_out >= B,
                 "subset_distance: bad shape (1 <= W <= %d, ldS >= W, 0 <= B < 2^31, "
                 "1 <= C < 2^24, ld_out >= B; W=%lld ldS=%lld B=%lld C=%lld ld_out=%lld)",
                 SS_MAX_W, (long long)W, (long long)ldS, (long long)B, (long long)C,
                 (long long)ld_out);
    ELFI_REQUIRE(metric >= ELFI_B200_METRIC_EUCLIDEAN && metric <= ELFI_B200_METRIC_CHEBYSHEV,
                 "subset_distance: metric code %d is not euclidean, sqeuclidean, cityblock or "
                 "chebyshev", int(metric));
    if (B == 0) return ELFI_B200_OK;
    return run_on_device(ctx, stream, [&](cudaStream_t s) {
        const int w = int(W), c = int(C);
        switch (metric) {
            case ELFI_B200_METRIC_EUCLIDEAN:
                return launch_subset_distance<ELFI_B200_METRIC_EUCLIDEAN>(
                    ctx, S, ldS, B, w, obs, ranges, comb, c, d_out, ld_out, s);
            case ELFI_B200_METRIC_SQEUCLIDEAN:
                return launch_subset_distance<ELFI_B200_METRIC_SQEUCLIDEAN>(
                    ctx, S, ldS, B, w, obs, ranges, comb, c, d_out, ld_out, s);
            case ELFI_B200_METRIC_CITYBLOCK:
                return launch_subset_distance<ELFI_B200_METRIC_CITYBLOCK>(
                    ctx, S, ldS, B, w, obs, ranges, comb, c, d_out, ld_out, s);
            default:
                return launch_subset_distance<ELFI_B200_METRIC_CHEBYSHEV>(
                    ctx, S, ldS, B, w, obs, ranges, comb, c, d_out, ld_out, s);
        }
    });
}

int elfi_b200_knn_entropy_f64(elfi_b200_ctx* ctx, const double* X, int64_t ldX, int64_t C,
                              int64_t n, int64_t q, int64_t k, double* R, double* logsum,
                              void* stream) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && X && R && logsum, "knn_entropy: NULL argument");
    ELFI_REQUIRE(q >= 1 && q <= KN_MAX_Q && ldX >= q && k >= 1 && k <= KN_MAX_K && n >= 1 &&
                     n <= ELFI_B200_KNN_MAX_N && C >= 1 && C <= ELFI_B200_KNN_MAX_SETS,
                 "knn_entropy: bad shape (1 <= q <= %d, ldX >= q, 1 <= k <= %d, 1 <= n <= 2^20, "
                 "1 <= C < 2^16; q=%lld ldX=%lld k=%lld n=%lld C=%lld)", KN_MAX_Q, KN_MAX_K,
                 (long long)q, (long long)ldX, (long long)k, (long long)n, (long long)C);
    return run_on_device(ctx, stream, [&](cudaStream_t s) {
        const dim3 grid(unsigned((n + KN_QUERIES - 1) / KN_QUERIES), unsigned(C));
        with_pow2<1, KN_MAX_K>(int(k), [&](auto kmax) {
            knn_radius_kernel<decltype(kmax)::value><<<grid, KN_QUERIES, 0, s>>>(
                X, ldX, int(n), int(q), int(k), R);
            return 0;
        });
        log_sum_kernel<<<unsigned(C), RED_THREADS, 0, s>>>(R, int(n), logsum);
        return ELFI_B200_OK;
    });
}

int elfi_b200_mrsse_f64(elfi_b200_ctx* ctx, const double* T, int64_t ldT, int64_t C, int64_t n,
                        int64_t q, const double* P, int64_t ldP, int64_t m, double* out,
                        void* stream) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && T && P && out, "mrsse: NULL argument");
    ELFI_REQUIRE(q >= 1 && q <= KN_MAX_Q && ldT >= q && ldP >= q && n >= 1 &&
                     n * q < (int64_t(1) << 31) && m >= 1 && m < (int64_t(1) << 31) && C >= 1 &&
                     C < (int64_t(1) << 31),
                 "mrsse: bad shape (1 <= q <= %d, ldT >= q, ldP >= q, 1 <= n q < 2^31, "
                 "1 <= m < 2^31, 1 <= C < 2^31; q=%lld ldT=%lld ldP=%lld n=%lld m=%lld C=%lld)",
                 KN_MAX_Q, (long long)q, (long long)ldT, (long long)ldP, (long long)n,
                 (long long)m, (long long)C);
    return run_on_device(ctx, stream, [&](cudaStream_t s) {
        mrsse_kernel<<<unsigned(C), RED_THREADS, 0, s>>>(T, ldT, n, int(q), P, ldP, m, out);
        return ELFI_B200_OK;
    });
}

}  // extern "C"
