// gnkstats.cu -- robust and octile summaries of the g-and-k examples on the device
// (elfi/examples/gnk.py:164-248, bignk.py), the bivariate g-and-k simulator (bignk.py:12-108) and
// the discrepancy euclidean_multiss (gnk.py:115-142).
//
// A summary needs 7 order-statistic pairs of a series (gnkstats.cuh), so one warp sorts a series
// with the bitonic networks of bitonic.cuh and lane 0 interpolates.  The fused simulators draw a
// row's observations straight into the sort registers: only the 4 or 7 summaries per dimension
// reach HBM instead of the (B, n_obs[, 2]) data matrix.
//
// Limits: series of 1 <= n <= 2048 (n <= 512 in registers, larger in shared memory); the fused
// simulators take n_obs <= 512.  NaN rules: see gnkstats.cuh (a NaN anywhere in a series makes
// all its octiles NaN).
#include "bitonic.cuh"
#include "boxmuller.cuh"
#include "common.cuh"
#include "gnkmath.cuh"
#include "gnkstats.cuh"
#include "leafsum.cuh"
#include "philox.cuh"
#include "rowquantiles.cuh"

namespace elfi {

constexpr uint32_t SALT_SIM_GNK = 0x474e4b30u;     // sim_gnk_kernel's stream (simulate.cu)
constexpr uint32_t SALT_SIM_BIGNK = 0x42474e4bu;   // one block per (row, observation)
constexpr int GNK_REGS_MAX = ELFI_B200_GNK_FUSED_MAX;
static_assert(GNK_REGS_MAX == 32 * 16, "the register sort holds 32 lanes x 16 keys");
constexpr int GNK_SERIES_MAX = ELFI_B200_GNK_SERIES_MAX;

// sort one series held in registers, then lane 0 writes its summary to out[j * step]
template <int KPL>
__device__ __forceinline__ void summarize_regs(uint64_t (&key)[KPL], int lane, int n, int kind,
                                               const GnkPicks& p, bool live, double* out, int step) {
    bitonic_in_registers<KPL>(key, lane);
    double a[GNK_NQ], b[GNK_NQ];
#pragma unroll
    for (int q = 0; q < GNK_NQ; ++q) {
        a[q] = u64_to_key(pick_reg(key, p.lo[q]));
        b[q] = u64_to_key(pick_reg(key, p.hi[q]));
    }
    const bool has_nan = pick_reg(key, n - 1) == ~uint64_t(0);
    if (live && lane == 0) gnk_summary(kind, p, a, b, has_nan, out, step);
}

// ---- summaries of a data matrix: series (row, dim) is X[row * ld_row + i * ld_obs + dim] ----
// One warp per series; the loop bounds are block-uniform so that the shuffles sit in convergent
// code (as in rowsort_regs_kernel).
template <int KPL>
__global__ void __launch_bounds__(256)
gnk_summaries_regs_kernel(const double* __restrict__ X, int64_t ld_row, int64_t ld_obs, int64_t B,
                          int n_, int d, int kind, GnkPicks p, double* __restrict__ out,
                          int64_t ld_out) {
    const int lane = threadIdx.x & 31;
    const int64_t S = B * d;
    for (int64_t base = int64_t(blockIdx.x) * 8; base < S; base += int64_t(gridDim.x) * 8) {
        const int64_t s = base + (threadIdx.x >> 5);
        const bool live = s < S;
        const int n = live ? n_ : 0;
        const int64_t row = live ? s / d : 0;
        const int dim = int(s - row * d) * int(live);
        const double* x = X + row * ld_row + dim;
        uint64_t key[KPL];
#pragma unroll
        for (int r = 0; r < KPL; ++r) {
            const int i = lane * KPL + r;
            key[r] = i < n ? key_to_u64(__ldg(x + int64_t(i) * ld_obs)) : ~uint64_t(0);
        }
        summarize_regs<KPL>(key, lane, n_, kind, p, live, out + row * ld_out + dim, d);
    }
}

__global__ void __launch_bounds__(256)
gnk_summaries_smem_kernel(const double* __restrict__ X, int64_t ld_row, int64_t ld_obs, int64_t B,
                          int n, int npow2, int d, int kind, GnkPicks p, double* __restrict__ out,
                          int64_t ld_out) {
    extern __shared__ uint64_t sk_all[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint64_t* sk = sk_all + size_t(warp) * npow2;
    const int64_t S = B * d;
    for (int64_t s = int64_t(blockIdx.x) * 8 + warp; s < S; s += int64_t(gridDim.x) * 8) {
        const int64_t row = s / d;
        const int dim = int(s - row * d);
        const double* x = X + row * ld_row + dim;
        for (int i = lane; i < npow2; i += 32)
            sk[i] = i < n ? key_to_u64(x[int64_t(i) * ld_obs]) : ~uint64_t(0);
        __syncwarp();
        bitonic_in_shared(sk, npow2, lane);
        if (lane == 0) {
            double a[GNK_NQ], b[GNK_NQ];
            for (int q = 0; q < GNK_NQ; ++q) {
                a[q] = u64_to_key(sk[p.lo[q]]);
                b[q] = u64_to_key(sk[p.hi[q]]);
            }
            gnk_summary(kind, p, a, b, sk[n - 1] == ~uint64_t(0), out + row * ld_out + dim, d);
        }
        __syncwarp();
    }
}

// ---- fused univariate simulator + summaries ---------------------------------------------------
// Lane L owns observations L*KPL .. L*KPL + KPL-1 (KPL even), i.e. the Philox blocks (row, pair)
// L*KPL/2 .. of sim_gnk_kernel, and evaluates the same gnk_quantile: the keys are the bits
// sim_gnk_kernel would have written.  At KPL 4 and 16 the register cap of two blocks per SM (128)
// spills the keys that live across the pow() calls to local memory, so those two take one block
// per SM; KPL 2 and 8 fit two.
template <int KPL>
__global__ void __launch_bounds__(256, (KPL == 4 || KPL == 16) ? 1 : 2)
sim_gnk_summaries_kernel(const double* __restrict__ A, const double* __restrict__ Bs,
                         const double* __restrict__ g, const double* __restrict__ k, double c,
                         int64_t B, int n_obs, uint64_t seed, uint64_t offset, int kind, GnkPicks p,
                         double* __restrict__ out, int64_t ld_out) {
    static_assert(KPL % 2 == 0, "observations are drawn in pairs");
    const int lane = threadIdx.x & 31;
    const Philox ph(seed);
    for (int64_t base = int64_t(blockIdx.x) * 8; base < B; base += int64_t(gridDim.x) * 8) {
        const int64_t i = base + (threadIdx.x >> 5);
        const bool live = i < B;
        const int n = live ? n_obs : 0;
        const double a = live ? A[i] : 0.0, b = live ? Bs[i] : 0.0;
        const double gg = live ? g[i] : 0.0, kk = live ? k[i] : 0.0;
        const uint64_t row = offset + uint64_t(i);
        uint64_t key[KPL];
#pragma unroll
        for (int r = 0; r < KPL; r += 2) {
            const int j = lane * KPL + r;
            key[r] = key[r + 1] = ~uint64_t(0);
            if (j < n) {
                double z0, z1;
                normal2(ph(uint32_t(row), uint32_t(row >> 32), uint32_t(j >> 1), SALT_SIM_GNK), z0, z1);
                key[r] = key_to_u64(gnk_quantile(a, b, gg, kk, c, z0));
                if (j + 1 < n) key[r + 1] = key_to_u64(gnk_quantile(a, b, gg, kk, c, z1));
            }
        }
        summarize_regs<KPL>(key, lane, n_obs, kind, p, live, out + i * ld_out, 1);
    }
}

// ---- bivariate g-and-k ------------------------------------------------------------------------
// Parameters P[row * ldP + 0..8] = A1, A2, B1, B2, g1, g2, k1, k2, rho (bignk.py's order).
// Observation j of a row: Philox block (row, j) -> n0, n1; z1 = n0, z2 = rho n0 + sqrt(1 - rho^2) n1
// (cov [[1, rho], [rho, 1]]); y_d = gnk_quantile(A_d, B_d, g_d, k_d, c, z_d).  |rho| > 1 (or NaN)
// makes both coordinates NaN.
struct BiGnkParams {
    double A0, A1, B0, B1, g0, g1, k0, k1, rho, sr;   // sr = sqrt(1 - rho^2)
};

__device__ __forceinline__ BiGnkParams bignk_params(const double* P) {
    BiGnkParams q;
    q.A0 = P[0]; q.A1 = P[1]; q.B0 = P[2]; q.B1 = P[3];
    q.g0 = P[4]; q.g1 = P[5]; q.k0 = P[6]; q.k1 = P[7]; q.rho = P[8];
    q.sr = __dsqrt_rn(__dsub_rn(1.0, __dmul_rn(q.rho, q.rho)));
    return q;
}

__device__ __forceinline__ void bignk_draw(const Philox& ph, uint64_t row, int j, const BiGnkParams& q,
                                           double c, double& y0, double& y1) {
    double n0, n1;
    normal2(ph(uint32_t(row), uint32_t(row >> 32), uint32_t(j), SALT_SIM_BIGNK), n0, n1);
    const double z0 = fabs(q.rho) <= 1.0 ? n0 : NAN;
    const double z1 = __dadd_rn(__dmul_rn(q.rho, n0), __dmul_rn(q.sr, n1));
    y0 = gnk_quantile(q.A0, q.B0, q.g0, q.k0, c, z0);
    y1 = gnk_quantile(q.A1, q.B1, q.g1, q.k1, c, z1);
}

// data (B, n_obs, 2): one thread per (row, observation)
__global__ void __launch_bounds__(256)
sim_bignk_kernel(const double* __restrict__ P, int64_t ldP, double c, int64_t B, int n_obs,
                 uint64_t seed, uint64_t offset, double* __restrict__ Y, int64_t ldY) {
    const int64_t total = B * n_obs;
    const Philox ph(seed);
    const bool vec = (ldY & 1) == 0 && (reinterpret_cast<uintptr_t>(Y) & 15) == 0;
    for (int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
         idx += int64_t(gridDim.x) * blockDim.x) {
        const int64_t i = idx / n_obs;
        const int j = int(idx - i * n_obs);
        const BiGnkParams q = bignk_params(P + i * ldP);
        double y0, y1;
        bignk_draw(ph, offset + uint64_t(i), j, q, c, y0, y1);
        double* dst = Y + i * ldY + 2 * j;
        if (vec) {
            *reinterpret_cast<double2*>(dst) = make_double2(y0, y1);
        } else {
            dst[0] = y0;
            dst[1] = y1;
        }
    }
}

// fused: one warp per row, two register series (one per coordinate)
template <int KPL>
__global__ void __launch_bounds__(256)
sim_bignk_summaries_kernel(const double* __restrict__ P, int64_t ldP, double c, int64_t B, int n_obs,
                           uint64_t seed, uint64_t offset, int kind, GnkPicks p,
                           double* __restrict__ out, int64_t ld_out) {
    const int lane = threadIdx.x & 31;
    const Philox ph(seed);
    for (int64_t base = int64_t(blockIdx.x) * 8; base < B; base += int64_t(gridDim.x) * 8) {
        const int64_t i = base + (threadIdx.x >> 5);
        const bool live = i < B;
        const int n = live ? n_obs : 0;
        const BiGnkParams q = bignk_params(P + (live ? i : 0) * ldP);
        const uint64_t row = offset + uint64_t(i);
        uint64_t key0[KPL], key1[KPL];
#pragma unroll
        for (int r = 0; r < KPL; ++r) {
            const int j = lane * KPL + r;
            key0[r] = key1[r] = ~uint64_t(0);
            if (j < n) {
                double y0, y1;
                bignk_draw(ph, row, j, q, c, y0, y1);
                key0[r] = key_to_u64(y0);
                key1[r] = key_to_u64(y1);
            }
        }
        summarize_regs<KPL>(key0, lane, n_obs, kind, p, live, out + i * ld_out, 2);
        summarize_regs<KPL>(key1, lane, n_obs, kind, p, live, out + i * ld_out + 1, 2);
    }
}

// ---- euclidean_multiss: sqrt(sum_j (S[i, j] - obs[j])^2), NumPy's pairwise order ---------------
template <int J>
__device__ __forceinline__ void push_sq(LeafSum& s, int j0, int K, const double* row,
                                        const double* obs) {
    const int j = j0 + J;
    if (j < K) {
        const double t = __dsub_rn(row[j], obs[j]);
        s.push<J>(j, __dmul_rn(t, t));
    }
    if constexpr (J + 1 < 8) push_sq<J + 1>(s, j0, K, row, obs);
}

__global__ void __launch_bounds__(256)
euclidean_multiss_kernel(const double* __restrict__ S, int64_t ldS, int64_t B, int K,
                         const double* __restrict__ obs, double* __restrict__ out) {
    const int64_t stride = int64_t(gridDim.x) * blockDim.x;
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < B; i += stride) {
        LeafSum s;
        s.begin(K);
        for (int j0 = 0; j0 < K; j0 += 8) push_sq<0>(s, j0, K, S + i * ldS, obs);
        out[i] = __dsqrt_rn(s.finish(K));
    }
}

// blocks of 8 warps, at most 8 per SM and at least one
static unsigned warp_blocks(const elfi_b200_ctx* ctx, int64_t warps) {
    const unsigned blocks = capped_grid(ctx, warps, 8, 8);
    return blocks < 1 ? 1 : blocks;
}

// picks_host: lo[7], hi[7], t[7] as doubles (ops.gnk_picks)
static int read_picks(const double* picks_host, int64_t n, GnkPicks* p) {
    ELFI_REQUIRE(picks_host != nullptr, "gnk summaries: picks are NULL");
    for (int q = 0; q < GNK_NQ; ++q) {
        const double lo = picks_host[q], hi = picks_host[GNK_NQ + q], t = picks_host[2 * GNK_NQ + q];
        ELFI_REQUIRE(lo >= 0 && lo < double(n) && hi >= 0 && hi < double(n) && lo == double(int(lo)) &&
                     hi == double(int(hi)) && t >= 0.0 && t <= 1.0,
                     "gnk summaries: pick %d (%g, %g, %g) invalid for n=%lld", q, lo, hi, t, (long long)n);
        p->lo[q] = int(lo);
        p->hi[q] = int(hi);
        p->t[q] = t;
    }
    return ELFI_B200_OK;
}

}  // namespace elfi

extern "C" {

int elfi_b200_gnk_summaries_f64(elfi_b200_ctx* ctx, const double* X, int64_t ld_row, int64_t ld_obs,
                                int64_t B, int64_t n, int64_t d, int32_t kind,
                                const double* picks_host, double* out, int64_t ld_out, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || (X && out)), "gnk_summaries: NULL argument");
    ELFI_REQUIRE(kind == GNK_ROBUST || kind == GNK_OCTILE, "gnk_summaries: unknown kind %d", kind);
    ELFI_REQUIRE(B >= 0 && n >= 1 && n <= GNK_SERIES_MAX && (d == 1 || d == 2),
                 "gnk_summaries: bad shape (1 <= n <= %d, d in {1, 2}; n=%lld d=%lld)", GNK_SERIES_MAX,
                 (long long)n, (long long)d);
    ELFI_REQUIRE(ld_obs >= d && ld_row >= (n - 1) * ld_obs + d && ld_out >= d * gnk_summary_width(kind),
                 "gnk_summaries: bad leading dimension");
    GnkPicks p;
    int rc = read_picks(picks_host, n, &p);
    if (rc) return rc;
    if (B == 0) return ELFI_B200_OK;
    const unsigned blocks = warp_blocks(ctx, B * d);
    const int ni = int(n), di = int(d);
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        if (n <= GNK_REGS_MAX) {
            with_pow2<1, 16>(kpl_for(ni, 1), [&](auto K) {
                gnk_summaries_regs_kernel<decltype(K)::value><<<blocks, 256, 0, stream>>>(
                    X, ld_row, ld_obs, B, ni, di, kind, p, out, ld_out);
            });
        } else {
            int npow2 = 2;
            while (npow2 < n) npow2 <<= 1;
            const size_t smem = size_t(8) * npow2 * 8;
            ELFI_CUDA_OK(cudaFuncSetAttribute(gnk_summaries_smem_kernel,
                                              cudaFuncAttributeMaxDynamicSharedMemorySize,
                                              int(smem)));
            gnk_summaries_smem_kernel<<<blocks, 256, smem, stream>>>(X, ld_row, ld_obs, B, ni, npow2,
                                                                     di, kind, p, out, ld_out);
        }
        return ELFI_B200_OK;
    });
}

int elfi_b200_sim_gnk_summaries_f64(elfi_b200_ctx* ctx, const double* A, const double* Bs,
                                    const double* g, const double* k, double c, int64_t B,
                                    int64_t n_obs, uint64_t seed, uint64_t offset, int32_t kind,
                                    const double* picks_host, double* out, int64_t ld_out,
                                    void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || (A && Bs && g && k && out)), "sim_gnk_summaries: NULL argument");
    ELFI_REQUIRE(kind == GNK_ROBUST || kind == GNK_OCTILE, "sim_gnk_summaries: unknown kind %d", kind);
    ELFI_REQUIRE(B >= 0 && n_obs >= 1 && n_obs <= GNK_REGS_MAX,
                 "sim_gnk_summaries: bad shape (1 <= n_obs <= %d; n_obs=%lld)", GNK_REGS_MAX,
                 (long long)n_obs);
    ELFI_REQUIRE(ld_out >= gnk_summary_width(kind), "sim_gnk_summaries: bad leading dimension");
    GnkPicks p;
    int rc = read_picks(picks_host, n_obs, &p);
    if (rc) return rc;
    if (B == 0) return ELFI_B200_OK;
    const unsigned blocks = warp_blocks(ctx, B);
    const int n = int(n_obs);
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        with_pow2<2, 16>(kpl_for(n, 2), [&](auto K) {
            sim_gnk_summaries_kernel<decltype(K)::value><<<blocks, 256, 0, stream>>>(
                A, Bs, g, k, c, B, n, seed, offset, kind, p, out, ld_out);
        });
        return ELFI_B200_OK;
    });
}

int elfi_b200_sim_bignk_f64(elfi_b200_ctx* ctx, const double* P, int64_t ldP, double c, int64_t B,
                            int64_t n_obs, uint64_t seed, uint64_t offset, double* Y, int64_t ldY,
                            int32_t kind, const double* picks_host, double* S, int64_t ldS,
                            void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || P), "sim_bignk: NULL argument");
    ELFI_REQUIRE(B >= 0 && n_obs >= 1 && n_obs < (int64_t(1) << 29) && ldP >= 9,
                 "sim_bignk: bad shape B=%lld n_obs=%lld ldP=%lld", (long long)B, (long long)n_obs,
                 (long long)ldP);
    ELFI_REQUIRE(Y == nullptr || ldY >= 2 * n_obs, "sim_bignk: bad leading dimension of the data");
    GnkPicks p;
    if (S) {
        ELFI_REQUIRE(kind == GNK_ROBUST || kind == GNK_OCTILE, "sim_bignk: unknown kind %d", kind);
        ELFI_REQUIRE(n_obs <= GNK_REGS_MAX, "sim_bignk: fused summaries need n_obs <= %d (n_obs=%lld)",
                     GNK_REGS_MAX, (long long)n_obs);
        ELFI_REQUIRE(ldS >= 2 * gnk_summary_width(kind), "sim_bignk: bad leading dimension of S");
        int rc = read_picks(picks_host, n_obs, &p);
        if (rc) return rc;
    }
    if (B == 0) return ELFI_B200_OK;
    const int n = int(n_obs);
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        if (Y)
            sim_bignk_kernel<<<capped_grid(ctx, B * n_obs, 256, 64), 256, 0, stream>>>(
                P, ldP, c, B, n, seed, offset, Y, ldY);
        if (S) {
            const unsigned blocks = warp_blocks(ctx, B);
            with_pow2<1, 16>(kpl_for(n, 1), [&](auto K) {
                sim_bignk_summaries_kernel<decltype(K)::value><<<blocks, 256, 0, stream>>>(
                    P, ldP, c, B, n, seed, offset, kind, p, S, ldS);
            });
        }
        return ELFI_B200_OK;
    });
}

int elfi_b200_euclidean_multiss_f64(elfi_b200_ctx* ctx, const double* S, int64_t ldS, int64_t B,
                                    int64_t K, const double* obs, double* out, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || (S && obs && out)), "euclidean_multiss: NULL argument");
    ELFI_REQUIRE(B >= 0 && K >= 1 && K <= LEAF_MAX_TERMS && ldS >= K,
                 "euclidean_multiss: bad shape (1 <= K <= %d; K=%lld)", LEAF_MAX_TERMS, (long long)K);
    if (B == 0) return ELFI_B200_OK;
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        euclidean_multiss_kernel<<<capped_grid(ctx, B, 256, 16), 256, 0, stream>>>(S, ldS, B, int(K),
                                                                                  obs, out);
        return ELFI_B200_OK;
    });
}

}  // extern "C"
