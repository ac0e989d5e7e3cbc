// ricker_wood.cu -- the 13 summary statistics of Wood (2010, Nature 466:1102) for the stochastic
// Ricker model, on any (B, n) matrix of counts on the device.  The host definition, and this
// project's reading of the paper (divisors, lags, no intercepts, the rank rule), is ss_wood in
// elfi_b200/examples/ricker.py; the contract is in include/elfi_b200.h.
//
// Columns: 0 mean, 1 number of zeros, 2..7 autocovariances at lags 0..5 (divisor n),
// 8..10 the cubic regression of the sorted differences on the sorted observed differences
// (coefficients = P e, P the 3 x (n-1) pseudo-inverse of the observed design, made on the host),
// 11..12 the autoregression y_{t+1}^0.3 = a1 y_t^0.3 + a2 y_t^0.6 (minimum-norm least squares).
//
// Layout: one warp per row, WOOD_WARPS warps per block.  A warp stages its row in shared memory
// (coalesced loads from any leading dimension), and
//   * lanes 0..5 each take the mean, then lane k the lag-k autocovariance, one term at a time in
//     NumPy's pairwise order (TreeSum: one leaf for n <= 128, the same tree above), so these seven
//     are NumPy's bits for every n <= 2048;
//   * the n-1 differences are sorted by the warp in shared memory (bitonic_in_shared, keys padded
//     to a power of two with the NaN key, which sorts last and is never read);
//   * the three dot products with P and the five sums of the 2 x 2 normal equations are lane-strided
//     partial sums closed by an xor butterfly: every lane ends with the same bits, and the order
//     depends only on n, so a row's result does not depend on B or on the call.
// Shared memory per warp: 16 result slots, the row (n doubles) and the keys (npow2(n - 1)): at most
// 4 x 4112 x 8 = 132 KiB per block at n = 2048.
#include "bitonic.cuh"
#include "common.cuh"
#include "treesum.cuh"

namespace elfi {

constexpr int WOOD_NOBS_MIN = ELFI_B200_RICKER_WOOD_NOBS_MIN;
// the shared-memory sort of gnk_summaries has the same bound
constexpr int WOOD_NOBS_MAX = ELFI_B200_RICKER_WOOD_NOBS_MAX;
constexpr int WOOD_WIDTH = ELFI_B200_RICKER_WOOD_WIDTH;
constexpr int WOOD_WARPS = 4;
constexpr int WOOD_LAGS = 6;          // autocovariances at lags 0 .. 5
constexpr int WOOD_SLOTS = 16;        // per-warp result slots (13 used)
using WoodSum = TreeSum<5>;
static_assert(WoodSum::max_terms() >= WOOD_NOBS_MAX, "TreeSum depth too small for WOOD_NOBS_MAX");

__host__ __device__ inline int wood_pow2(int m) {
    int p = 8;
    while (p < m) p <<= 1;
    return p;
}

inline size_t wood_warp_doubles(int n) { return size_t(WOOD_SLOTS) + n + wood_pow2(n - 1); }

// s.push of the terms j0 .. j0 + 7 (those below m) of f, K = j % 8 known at compile time
template <int J, class F>
__device__ __forceinline__ void wood_push8(WoodSum& s, int j0, int m, const F& f) {
    if (j0 + J < m) s.push<J>(j0 + J, f(j0 + J));
    if constexpr (J + 1 < 8) wood_push8<J + 1>(s, j0, m, f);
}
template <int J, class F>
__device__ __forceinline__ void wood_mid8(WoodSum& s, int j0, const F& f) {
    s.push_mid<J>(f(j0 + J));
    if constexpr (J + 1 < 8) wood_mid8<J + 1>(s, j0, f);
}

// sum_{j < m} f(j) in NumPy's pairwise order (np.add.reduce over a contiguous run of m terms)
template <class F>
__device__ double wood_pairwise(int m, const F& f) {
    WoodSum s;
    s.begin(m);
    for (int j0 = 0; j0 < m; j0 += 8) {
        if (s.all_mid(j0, j0 + 7))
            wood_mid8<0>(s, j0, f);
        else
            wood_push8<0>(s, j0, m, f);
    }
    return s.finish(m);
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
    return v;
}

__global__ void __launch_bounds__(WOOD_WARPS * 32)
ricker_wood_kernel(const double* __restrict__ Y, int64_t ldY, int64_t B, int n,
                   const double* __restrict__ P, double* __restrict__ out, int64_t ld_out) {
    extern __shared__ double wood_smem[];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int npow2 = wood_pow2(n - 1);
    double* res = wood_smem + size_t(warp) * (WOOD_SLOTS + n + npow2);
    double* ys = res + WOOD_SLOTS;
    uint64_t* keys = reinterpret_cast<uint64_t*>(ys + n);
    const int nd = n - 1;   // differences, regression rows
    for (int64_t row = int64_t(blockIdx.x) * WOOD_WARPS + warp; row < B;
         row += int64_t(gridDim.x) * WOOD_WARPS) {
        const double* y = Y + row * ldY;
        double* o = out + row * ld_out;
        bool bad = false;
        unsigned zeros = 0;
        for (int j = lane; j < n; j += 32) {
            const double v = y[j];
            ys[j] = v;
            bad |= !isfinite(v);
            zeros += (v == 0.0) ? 1u : 0u;
        }
        if (__any_sync(0xffffffffu, bad)) {
            if (lane < WOOD_WIDTH) o[lane] = __longlong_as_double(0x7ff8000000000000LL);
            continue;
        }
        zeros = __reduce_add_sync(0xffffffffu, zeros);
        __syncwarp();

        // keys of the differences; the first nonzero y_t (t < n - 1) of the rank rule
        for (int t = lane; t < npow2; t += 32)
            keys[t] = t < nd ? key_to_u64(__dsub_rn(ys[t + 1], ys[t])) : ~uint64_t(0);
        int first = -1;
        for (int t0 = 0; t0 < nd && first < 0; t0 += 32) {
            const unsigned nz = __ballot_sync(0xffffffffu, t0 + lane < nd && ys[t0 + lane] != 0.0);
            if (nz) first = t0 + __ffs(nz) - 1;
        }

        // the autoregression's sums: [u v]' [u v], [u v]' w, and w over the t with y_t = k
        double suu = 0.0, suv = 0.0, svv = 0.0, suw = 0.0, svw = 0.0, skw = 0.0, nk = 0.0;
        bool other = false;
        if (first >= 0) {
            const double k = ys[first];
            for (int t = lane; t < nd; t += 32) {
                const double yt = ys[t];
                const double u = pow(yt, 0.3), v = pow(yt, 0.6), w = pow(ys[t + 1], 0.3);
                suu += u * u;
                suv += u * v;
                svv += v * v;
                suw += u * w;
                svw += v * w;
                if (yt == k) {
                    skw += w;
                    nk += 1.0;
                }
                other |= yt != 0.0 && yt != k;
            }
        }
        other = __any_sync(0xffffffffu, other);
        suu = warp_sum(suu);
        suv = warp_sum(suv);
        svv = warp_sum(svv);
        suw = warp_sum(suw);
        svw = warp_sum(svw);
        skw = warp_sum(skw);
        nk = warp_sum(nk);

        __syncwarp();
        bitonic_in_shared(keys, npow2, lane);
        double c0 = 0.0, c1 = 0.0, c2 = 0.0;
        for (int t = lane; t < nd; t += 32) {
            const double e = u64_to_key(keys[t]);
            c0 += __ldg(P + t) * e;
            c1 += __ldg(P + nd + t) * e;
            c2 += __ldg(P + 2 * nd + t) * e;
        }
        c0 = warp_sum(c0);
        c1 = warp_sum(c1);
        c2 = warp_sum(c2);

        if (lane < WOOD_LAGS) {
            // pass 0: the mean (every one of these lanes); pass 1: the autocovariance at lag = lane
            const double* x = ys;
            const int lag = lane;
            double mean = 0.0;
#pragma unroll 1
            for (int pass = 0; pass < 2; ++pass) {
                const double sum = wood_pairwise(pass ? n - lag : n, [x, mean, lag, pass](int j) {
                    return pass ? __dmul_rn(__dsub_rn(x[j], mean), __dsub_rn(x[j + lag], mean)) : x[j];
                });
                if (pass)
                    res[2 + lag] = __ddiv_rn(sum, double(n));
                else
                    mean = __ddiv_rn(sum, double(n));
            }
            if (lane == 0) res[0] = mean;
        }
        if (lane == 0) {
            double a1 = 0.0, a2 = 0.0;
            if (first >= 0 && !other) {          // one distinct nonzero value k: proportional columns
                const double k = ys[first];
                const double s = skw / nk;
                const double k3 = pow(k, 0.3), k6 = pow(k, 0.6);
                const double den = k6 + pow(k, 1.2);
                a1 = s * k3 / den;
                a2 = s * k6 / den;
            } else if (first >= 0) {             // full column rank: the normal equations
                const double det = suu * svv - suv * suv;
                a1 = (svv * suw - suv * svw) / det;
                a2 = (suu * svw - suv * suw) / det;
            }
            res[1] = double(zeros);
            res[8] = c0;
            res[9] = c1;
            res[10] = c2;
            res[11] = a1;
            res[12] = a2;
        }
        __syncwarp();
        if (lane < WOOD_WIDTH) o[lane] = res[lane];
        __syncwarp();   // the next row overwrites ys, keys and res
    }
}

}  // namespace elfi

extern "C" {

int elfi_b200_ricker_wood_f64(elfi_b200_ctx* ctx, const double* Y, int64_t ldY, int64_t B, int64_t n,
                              const double* P, double* out, int64_t ld_out, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || (Y && P && out)), "ricker_wood: NULL argument");
    ELFI_REQUIRE(B >= 0 && n >= WOOD_NOBS_MIN && n <= WOOD_NOBS_MAX && ldY >= n &&
                     ld_out >= WOOD_WIDTH,
                 "ricker_wood: bad shape (%d <= n <= %d, ldY >= n, ld_out >= %d; B=%lld n=%lld "
                 "ldY=%lld ld_out=%lld)", WOOD_NOBS_MIN, WOOD_NOBS_MAX, WOOD_WIDTH, (long long)B,
                 (long long)n, (long long)ldY, (long long)ld_out);
    if (B == 0) return ELFI_B200_OK;
    const size_t smem = WOOD_WARPS * wood_warp_doubles(int(n)) * sizeof(double);
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        ELFI_CUDA_OK(cudaFuncSetAttribute(
            ricker_wood_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
            int(WOOD_WARPS * wood_warp_doubles(WOOD_NOBS_MAX) * sizeof(double))));
        ricker_wood_kernel<<<capped_grid(ctx, B, WOOD_WARPS, 16), WOOD_WARPS * 32, smem, stream>>>(
            Y, ldY, B, int(n), P, out, ld_out);
        return ELFI_B200_OK;
    });
}

}  // extern "C"
