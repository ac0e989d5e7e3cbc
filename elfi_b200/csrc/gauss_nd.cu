// gauss_nd.cu -- the n-D Gaussian mean model of elfi/examples/gauss.py (nd_mean=True): the axis-1
// mean and variance of (B, n, D) data, the reference's euclidean_multidim distance, and the
// throughput-mode multivariate normal simulator with the summaries fused.
//
// NumPy's orders (np.mean / np.var(y, axis=1) of a C-contiguous (B, n, D) array):
//   D = 1   the axis of length 1 is dropped and each row is one pairwise sum over the n
//           observations (pairwise.cuh), as ops.meanvar;
//   D >= 2  each coordinate is a plain left fold over t = 0 .. n - 1.
// Both start from 0.0 (np.add.reduce's identity: a row of -0.0 sums to +0.0).  The variance is
// sum_t (y - m) * (y - m) in the same order, m = sum / n, then divided by n.  The distance sums
// its D squared differences of a contiguous (B, D) array, i.e. one pairwise sum per row.
//
// Random streams (Philox4x32-10 keyed by the seed; counter (row, row >> 32, q / 2, SALT_GAUSS_ND)),
// row = offset + i: the row's normals are numbered q = t D + k (observation t, coordinate k), and
// block q / 2 gives normals 2 (q / 2) and 2 (q / 2) + 1 (boxmuller.cuh, n0 then n1).  No normal is
// skipped, also for odd D, and every value is a pure function of (seed, offset + row, q).
//
// Simulator layout: one thread per row, D a template parameter so that the means, the normals of
// one observation and the D running sums are registers, and the factor A (D x D, at most 2 KiB) is a
// kernel parameter: every thread of a warp reads the same A[k][j] at a compile-time offset, so the
// FMAs take it straight from the constant bank.  For D >= 2 the variance needs the final mean of
// every coordinate before its second sum, so the second pass regenerates the row from its stream:
// keeping it on chip would take n_obs D 8 bytes per row (6.4 KiB at n_obs = 50, D = 16), i.e. at
// most one warp of rows per SM in shared memory, where the regenerating kernel keeps 16 warps busy.
// The data, when asked for, is written in the first pass only.
#include "boxmuller.cuh"
#include "common.cuh"
#include "pairwise.cuh"
#include "philox.cuh"

namespace elfi {

constexpr uint32_t SALT_GAUSS_ND = 0x47534e44u;   // "GSND"
constexpr int GND_THREADS = 128;
constexpr int GND_D_MAX = ELFI_B200_GAUSS_ND_D_MAX;
constexpr int64_t GND_NOBS_MAX = ELFI_B200_GAUSS_ND_NOBS_MAX;
constexpr int64_t GND_SUMM_NOBS_MAX = ELFI_B200_GAUSS_ND_SUMM_NOBS_MAX;
constexpr int64_t GND_BATCH_MAX = int64_t(0x7fffffff) * GND_THREADS;   // one row per thread
static_assert(GND_NOBS_MAX <= PairwiseStream<6>::max_terms(), "the D = 1 simulator sums one row "
              "with a pairwise stack of depth 6");
static_assert(GND_SUMM_NOBS_MAX <= PairwiseStream<24>::max_terms(), "summary rows fit depth 24");

// the factor of the covariance, row-major A[k * GND_D_MAX + j]; passed by value
struct GaussNdFactor {
    double a[GND_D_MAX * GND_D_MAX];
};

// sum_{j < m} term(j) in NumPy's pairwise order, from 0.0
template <int MAXD, class Term>
__device__ __forceinline__ double pairwise_row(PairwiseStream<MAXD>& pw, int m, Term term) {
    double buf[8];
    pw.begin(m);
    for (int j0 = 0; j0 < m; j0 += 8) {
        const int cnt = (m - j0) < 8 ? (m - j0) : 8;
#pragma unroll
        for (int k = 0; k < 8; ++k) buf[k] = k < cnt ? term(j0 + k) : 0.0;
        pw.feed8(j0, buf, cnt);
    }
    return __dadd_rn(0.0, pw.finish());
}

__device__ __forceinline__ double sq_dev(double y, double m) {
    const double c = __dsub_rn(y, m);
    return __dmul_rn(c, c);
}

// ---- summaries of (B, n, D) data: one thread per (row, coordinate) -------------------------------
template <bool PAIRWISE>
__global__ void __launch_bounds__(GND_THREADS)
gauss_nd_summaries_kernel(const double* __restrict__ X, int64_t ld_b, int64_t ld_t, int64_t ld_j,
                          int64_t B, int n, int64_t D, double* __restrict__ out, int64_t ld_out) {
    const int64_t idx = int64_t(blockIdx.x) * GND_THREADS + threadIdx.x;
    if (idx >= B * D) return;
    const int64_t b = idx / D, j = idx - b * D;
    const double* x = X + b * ld_b + j * ld_j;
    double mean, ss;
    if constexpr (PAIRWISE) {
        PairwiseStream<24> pw;
        mean = pairwise_row(pw, n, [&](int t) { return __ldg(x + t * ld_t); }) / double(n);
        ss = pairwise_row(pw, n, [&](int t) { return sq_dev(__ldg(x + t * ld_t), mean); });
    } else {
        double s = 0.0;
        for (int t = 0; t < n; ++t) s = __dadd_rn(s, __ldg(x + t * ld_t));
        mean = s / double(n);
        ss = 0.0;
        for (int t = 0; t < n; ++t) ss = __dadd_rn(ss, sq_dev(__ldg(x + t * ld_t), mean));
    }
    out[b * ld_out + j] = mean;
    out[b * ld_out + D + j] = ss / double(n);
}

// ---- euclidean_multidim: one thread per row -------------------------------------------------------
__global__ void __launch_bounds__(GND_THREADS)
gauss_nd_distance_kernel(const double* __restrict__ S, int64_t ld_b, int64_t ld_j, int64_t B, int D,
                         const double* __restrict__ obs, double* __restrict__ d) {
    const int64_t b = int64_t(blockIdx.x) * GND_THREADS + threadIdx.x;
    if (b >= B) return;
    const double* s = S + b * ld_b;
    PairwiseStream<24> pw;
    d[b] = sqrt(pairwise_row(pw, D, [&](int j) { return sq_dev(__ldg(s + j * ld_j), __ldg(obs + j)); }));
}

// ---- simulator ------------------------------------------------------------------------------------
// observation y_j = (z_0 A_0j + sum_{k >= 1} z_k A_kj, by FMA in ascending k) + mu_j
template <int D>
__device__ __forceinline__ double gnd_coord(const double (&z)[D], const GaussNdFactor& A, int j,
                                            double mu) {
    double s = __dmul_rn(z[0], A.a[j]);
#pragma unroll
    for (int k = 1; k < D; ++k) s = __fma_rn(z[k], A.a[k * GND_D_MAX + j], s);
    return __dadd_rn(s, mu);
}

// D = 1: eight observations per step (four Philox blocks), summed by a pairwise stream.
template <bool WRITE_Y>
__global__ void __launch_bounds__(GND_THREADS)
sim_gauss_nd1_kernel(const double* __restrict__ mu, int64_t ld_b, int64_t B, GaussNdFactor A,
                     int n_obs, uint64_t seed, uint64_t offset, double* __restrict__ Y,
                     int64_t ldY, double* __restrict__ S, int64_t ldS) {
    const int64_t i = int64_t(blockIdx.x) * GND_THREADS + threadIdx.x;
    if (i >= B) return;
    const Philox ph(seed);
    const uint64_t row = offset + uint64_t(i);
    const uint32_t r0 = uint32_t(row), r1 = uint32_t(row >> 32);
    const double m = mu[i * ld_b];
    PairwiseStream<6> pw;
    double mean = 0.0;
    for (int pass = 0; pass < (S ? 2 : 1); ++pass) {
        if (S) pw.begin(n_obs);
        for (int k0 = 0; k0 < n_obs; k0 += 8) {
            double y[8];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                double z[1], z1[1];
                normal2(ph(r0, r1, uint32_t((k0 >> 1) + q), SALT_GAUSS_ND), z[0], z1[0]);
                y[2 * q] = gnd_coord<1>(z, A, 0, m);
                y[2 * q + 1] = gnd_coord<1>(z1, A, 0, m);
            }
            const int cnt = (n_obs - k0) < 8 ? (n_obs - k0) : 8;
            if (WRITE_Y && pass == 0) {
#pragma unroll
                for (int e = 0; e < 8; ++e)
                    if (e < cnt) Y[i * ldY + k0 + e] = y[e];
            }
            if (S) {
                double t[8];
#pragma unroll
                for (int e = 0; e < 8; ++e) t[e] = pass == 0 ? y[e] : sq_dev(y[e], mean);
                pw.feed8(k0, t, cnt);
            }
        }
        if (S) {
            const double v = __dadd_rn(0.0, pw.finish()) / double(n_obs);
            if (pass == 0) { mean = v; S[i * ldS] = v; } else { S[i * ldS + 1] = v; }
        }
    }
}

// D >= 2: one sweep over the row's observations, acc[j] += y_j (SQ false) or (y_j - mean_j)^2 (SQ
// true) as a left fold over t; the data is written when y_out is not NULL.
template <int D, bool SQ>
__device__ __forceinline__ void gnd_sweep(const Philox& ph, uint32_t r0, uint32_t r1,
                                          const GaussNdFactor& A, const double (&m)[D],
                                          const double (&mean)[D], double (&acc)[D], int n_obs,
                                          double* __restrict__ y_out) {
#pragma unroll
    for (int j = 0; j < D; ++j) acc[j] = 0.0;
    double spare = 0.0;   // the second normal of the last block, for an odd normal index q
    for (int t = 0; t < n_obs; ++t) {
        const uint32_t q0 = uint32_t(t) * uint32_t(D);
        double z[D];
#pragma unroll
        for (int k = 0; k < D; ++k) {
            const uint32_t q = q0 + uint32_t(k);
            // with D even, q and k have the same parity
            const bool even = (D % 2 == 0) ? (k % 2 == 0) : ((q & 1u) == 0u);
            if (even)
                normal2(ph(r0, r1, q >> 1, SALT_GAUSS_ND), z[k], spare);
            else
                z[k] = spare;
        }
#pragma unroll
        for (int j = 0; j < D; ++j) {
            const double y = gnd_coord<D>(z, A, j, m[j]);
            if (y_out) y_out[q0 + j] = y;
            acc[j] = __dadd_rn(acc[j], SQ ? sq_dev(y, mean[j]) : y);
        }
    }
}

// D >= 2: the first sweep writes the data and sums the means, the second regenerates the row and
// sums the squared deviations.
template <int D, bool WRITE_Y>
__global__ void __launch_bounds__(GND_THREADS)
sim_gauss_nd_kernel(const double* __restrict__ mu, int64_t ld_b, int64_t ld_j, int64_t B,
                    GaussNdFactor A, int n_obs, uint64_t seed, uint64_t offset,
                    double* __restrict__ Y, int64_t ldY, double* __restrict__ S, int64_t ldS) {
    const int64_t i = int64_t(blockIdx.x) * GND_THREADS + threadIdx.x;
    if (i >= B) return;
    const Philox ph(seed);
    const uint64_t row = offset + uint64_t(i);
    const uint32_t r0 = uint32_t(row), r1 = uint32_t(row >> 32);
    double m[D], acc[D], mean[D];
#pragma unroll
    for (int j = 0; j < D; ++j) {
        m[j] = mu[i * ld_b + j * ld_j];
        mean[j] = 0.0;
    }
    gnd_sweep<D, false>(ph, r0, r1, A, m, mean, acc, n_obs, WRITE_Y ? Y + i * ldY : nullptr);
    if (!S) return;
#pragma unroll
    for (int j = 0; j < D; ++j) {
        mean[j] = acc[j] / double(n_obs);
        S[i * ldS + j] = mean[j];
    }
    gnd_sweep<D, true>(ph, r0, r1, A, m, mean, acc, n_obs, nullptr);
#pragma unroll
    for (int j = 0; j < D; ++j) S[i * ldS + D + j] = acc[j] / double(n_obs);
}

template <int D>
static void sim_gauss_nd_launch(unsigned blocks, cudaStream_t stream, const double* mu, int64_t ld_b,
                                int64_t ld_j, int64_t B, const GaussNdFactor& A, int n_obs,
                                uint64_t seed, uint64_t offset, double* Y, int64_t ldY, double* S,
                                int64_t ldS) {
    if (Y)
        sim_gauss_nd_kernel<D, true><<<blocks, GND_THREADS, 0, stream>>>(
            mu, ld_b, ld_j, B, A, n_obs, seed, offset, Y, ldY, S, ldS);
    else
        sim_gauss_nd_kernel<D, false><<<blocks, GND_THREADS, 0, stream>>>(
            mu, ld_b, ld_j, B, A, n_obs, seed, offset, Y, ldY, S, ldS);
}

template <int D>
static void sim_gauss_nd_dispatch(int d, unsigned blocks, cudaStream_t stream, const double* mu,
                                  int64_t ld_b, int64_t ld_j, int64_t B, const GaussNdFactor& A,
                                  int n_obs, uint64_t seed, uint64_t offset, double* Y, int64_t ldY,
                                  double* S, int64_t ldS) {
    if (d == D) {
        sim_gauss_nd_launch<D>(blocks, stream, mu, ld_b, ld_j, B, A, n_obs, seed, offset, Y, ldY, S,
                               ldS);
        return;
    }
    if constexpr (D < GND_D_MAX)
        sim_gauss_nd_dispatch<D + 1>(d, blocks, stream, mu, ld_b, ld_j, B, A, n_obs, seed, offset, Y,
                                     ldY, S, ldS);
}

}  // namespace elfi

extern "C" {

int elfi_b200_gauss_nd_summaries_f64(elfi_b200_ctx* ctx, const double* X, int64_t ld_b,
                                     int64_t ld_t, int64_t ld_j, int64_t B, int64_t n, int64_t D,
                                     double* out, int64_t ld_out, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || (X && out)), "gauss_nd_summaries: NULL argument");
    ELFI_REQUIRE(B >= 0 && n >= 1 && n <= GND_SUMM_NOBS_MAX && D >= 1 &&
                     (B == 0 || D <= (int64_t(1) << 62) / B) && ld_out >= 2 * D,
                 "gauss_nd_summaries: bad shape (1 <= n <= %lld, D >= 1, ld_out >= 2 D; B=%lld "
                 "n=%lld D=%lld ld_out=%lld)", (long long)GND_SUMM_NOBS_MAX, (long long)B,
                 (long long)n, (long long)D, (long long)ld_out);
    if (B == 0) return ELFI_B200_OK;
    const int64_t blocks = (B * D + GND_THREADS - 1) / GND_THREADS;
    ELFI_REQUIRE(blocks <= 0x7fffffff, "gauss_nd_summaries: B * D = %lld too large",
                 (long long)(B * D));
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        if (D == 1)
            gauss_nd_summaries_kernel<true><<<unsigned(blocks), GND_THREADS, 0, stream>>>(
                X, ld_b, ld_t, ld_j, B, int(n), D, out, ld_out);
        else
            gauss_nd_summaries_kernel<false><<<unsigned(blocks), GND_THREADS, 0, stream>>>(
                X, ld_b, ld_t, ld_j, B, int(n), D, out, ld_out);
        ELFI_CUDA_OK(cudaGetLastError());
        return ELFI_B200_OK;
    });
}

int elfi_b200_gauss_nd_distance_f64(elfi_b200_ctx* ctx, const double* S, int64_t ld_b,
                                    int64_t ld_j, int64_t B, int64_t D, const double* obs,
                                    double* d, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || (S && obs && d)), "gauss_nd_distance: NULL argument");
    ELFI_REQUIRE(B >= 0 && D >= 1 && D <= GND_SUMM_NOBS_MAX && B <= GND_BATCH_MAX,
                 "gauss_nd_distance: bad shape (1 <= D <= %lld; B=%lld D=%lld)",
                 (long long)GND_SUMM_NOBS_MAX, (long long)B, (long long)D);
    if (B == 0) return ELFI_B200_OK;
    const unsigned blocks = unsigned((B + GND_THREADS - 1) / GND_THREADS);
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        gauss_nd_distance_kernel<<<blocks, GND_THREADS, 0, stream>>>(S, ld_b, ld_j, B, int(D), obs,
                                                                     d);
        ELFI_CUDA_OK(cudaGetLastError());
        return ELFI_B200_OK;
    });
}

int elfi_b200_sim_gauss_nd_f64(elfi_b200_ctx* ctx, const double* mu, int64_t ld_b, int64_t ld_j,
                               int64_t B, int64_t D, const double* A_host, int64_t n_obs,
                               uint64_t seed, uint64_t offset, double* Y, int64_t ldY, double* S,
                               int64_t ldS, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && A_host && (B == 0 || mu), "sim_gauss_nd: NULL argument");
    ELFI_REQUIRE(B >= 0 && B <= GND_BATCH_MAX && D >= 1 && D <= GND_D_MAX && n_obs >= 1 &&
                     n_obs <= GND_NOBS_MAX,
                 "sim_gauss_nd: bad shape (1 <= D <= %d, 1 <= n_obs <= %lld; B=%lld D=%lld "
                 "n_obs=%lld)", GND_D_MAX, (long long)GND_NOBS_MAX, (long long)B, (long long)D,
                 (long long)n_obs);
    ELFI_REQUIRE(Y || S, "sim_gauss_nd: nothing to produce (Y and S are both NULL)");
    ELFI_REQUIRE((!Y || ldY >= n_obs * D) && (!S || ldS >= 2 * D),
                 "sim_gauss_nd: bad leading dimension (ldY >= n_obs D, ldS >= 2 D; ldY=%lld "
                 "ldS=%lld)", (long long)ldY, (long long)ldS);
    if (B == 0) return ELFI_B200_OK;
    GaussNdFactor A;
    for (int k = 0; k < GND_D_MAX * GND_D_MAX; ++k) A.a[k] = 0.0;
    for (int64_t k = 0; k < D; ++k)
        for (int64_t j = 0; j < D; ++j) A.a[k * GND_D_MAX + j] = A_host[k * D + j];
    const unsigned blocks = unsigned((B + GND_THREADS - 1) / GND_THREADS);
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        if (D == 1) {
            if (Y)
                sim_gauss_nd1_kernel<true><<<blocks, GND_THREADS, 0, stream>>>(
                    mu, ld_b, B, A, int(n_obs), seed, offset, Y, ldY, S, ldS);
            else
                sim_gauss_nd1_kernel<false><<<blocks, GND_THREADS, 0, stream>>>(
                    mu, ld_b, B, A, int(n_obs), seed, offset, Y, ldY, S, ldS);
        } else {
            sim_gauss_nd_dispatch<2>(int(D), blocks, stream, mu, ld_b, ld_j, B, A, int(n_obs), seed,
                                     offset, Y, ldY, S, ldS);
        }
        ELFI_CUDA_OK(cudaGetLastError());
        return ELFI_B200_OK;
    });
}

}  // extern "C"
