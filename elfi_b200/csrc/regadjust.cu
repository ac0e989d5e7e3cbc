// regadjust.cu -- the local-linear regression adjustment of Beaumont et al. (2002)
// (elfi/methods/post_processing.py: LinearAdjustment) for N rows of q summaries S, the observed
// summaries o and p parameters T.  The regressors are x_i = S_i - o; a group is a set of rows and
// the parameter columns fitted on them.
//
// Entry points and their launches, in stream order:
//   mask:    regadj_mask_kernel: flags[i] = every S[i, j] - o[j] is finite, and per parameter k the
//            count of flagged rows whose T[i, k] is not finite (integer atomics: exact counts).
//   moments: regadj_colsum_kernel (one CTA per chunk) and regadj_mean_kernel: n_g and the means of
//            [S - o | T_g] over the group's rows; regadj_cross_kernel (one CTA per chunk and 64 x 64
//            lower tile): the chunk's centred cross-products; regadj_cross_reduce_kernel: the left
//            fold over the chunk sums, mirrored to a full symmetric matrix.
//   adjust:  regadj_adjust_kernel writes T[i, k] - sum_j (S[i, j] - o_j) coef[j, k] for the group's
//            rows in row order: at index i when every row is in the group, otherwise at the row's
//            rank among the group's rows (regadj_count_kernel and regadj_scan_kernel give each
//            CTA's first rank).
//
// Determinism: the chunk length depends on N and d = q + p_g only (ra_chunks), never on the GPU.
// Each chunk sum starts from zero, rows are added in row order within a chunk, and the chunk sums
// are added left to right, so the moments are a function of the rows alone: the same bits on every
// run and on any SM count.  No floating-point atomics.
//
// The cross-product runs on plain FP64 FMA with a 4 x 4 register tile per thread (DESIGN.md §7,
// "Regression adjustment", gives the reason).
#include <cmath>

#include "common.cuh"

namespace elfi {

constexpr int RA_D_MAX = ELFI_B200_REGADJ_D_MAX;
constexpr int RA_THREADS = 256;
constexpr int RA_TILE = 64;                  // lower tiles of the cross-product
constexpr int RA_SLAB = 32;                  // rows staged in shared memory per step
constexpr int64_t RA_MIN_CHUNK = 256;        // fewest rows of a chunk
constexpr int64_t RA_CTA_BUDGET = 2048;      // chunk x tile CTAs of the cross-product stage
constexpr int RA_ADJ_ROWS = 8 * RA_THREADS;  // rows of one CTA of the adjust stage

// one group: the regressors S - o, the parameter columns cols[0 .. pg - 1] of T, and the rows
// flags[i] != 0 with (sel < 0 or T[i, sel] finite)
struct RaGroup {
    const double* S;
    int64_t ldS;
    const double* o;
    const double* T;
    int64_t ldT;
    const uint8_t* flags;
    const int32_t* cols;
    int q;
    int pg;
    int sel;
};

__device__ __forceinline__ bool ra_member(const RaGroup& g, int64_t i) {
    return g.flags[i] && (g.sel < 0 || isfinite(g.T[i * g.ldT + g.sel]));
}

// column j of [S - o | T_g] at row i
__device__ __forceinline__ double ra_value(const RaGroup& g, int64_t i, int j) {
    return j < g.q ? g.S[i * g.ldS + j] - g.o[j] : g.T[i * g.ldT + g.cols[j - g.q]];
}

struct RaChunks {
    int64_t rows;    // rows per chunk, a multiple of RA_SLAB
    int64_t n;       // chunks
    int tiles;       // 64 x 64 lower tiles of the d x d cross-product
};

// the chunking of the moment stages: a function of N and d alone
static RaChunks ra_chunks(int64_t N, int d) {
    RaChunks c;
    const int t = (d + RA_TILE - 1) / RA_TILE;
    c.tiles = t * (t + 1) / 2;
    const int64_t target = RA_CTA_BUDGET / c.tiles > 1 ? RA_CTA_BUDGET / c.tiles : 1;
    int64_t rows = (N + target - 1) / target;
    rows = (rows + RA_SLAB - 1) / RA_SLAB * RA_SLAB;
    c.rows = rows > RA_MIN_CHUNK ? rows : RA_MIN_CHUNK;
    c.n = (N + c.rows - 1) / c.rows;
    return c;
}

__global__ void __launch_bounds__(RA_THREADS)
regadj_mask_kernel(const double* __restrict__ S, int64_t ldS, int64_t N, int q,
                   const double* __restrict__ o, const double* __restrict__ T, int64_t ldT, int p,
                   uint8_t* __restrict__ flags, unsigned long long* __restrict__ counts) {
    __shared__ unsigned int cnt[RA_D_MAX + 1];
    for (int k = threadIdx.x; k <= p; k += RA_THREADS) cnt[k] = 0;
    __syncthreads();
    const int64_t stride = int64_t(gridDim.x) * RA_THREADS;
    for (int64_t base = int64_t(blockIdx.x) * RA_THREADS; base < N; base += stride) {
        const int64_t i = base + threadIdx.x;
        bool ok = false;
        if (i < N) {
            const double* row = S + i * ldS;
            ok = true;
            for (int j = 0; j < q; ++j) ok &= bool(isfinite(row[j] - o[j]));
            flags[i] = ok;
            if (ok) {
                const double* t = T + i * ldT;
                for (int k = 0; k < p; ++k)
                    if (!isfinite(t[k])) atomicAdd(&cnt[1 + k], 1u);
            }
        }
        const int c = __syncthreads_count(ok);
        if (threadIdx.x == 0) cnt[0] += unsigned(c);
    }
    __syncthreads();
    for (int k = threadIdx.x; k <= p; k += RA_THREADS)
        if (cnt[k]) atomicAdd(&counts[k], (unsigned long long)cnt[k]);
}

// psum[c * d + j] = sum of column j over the group's rows of chunk c, pcount[c] their number.
// W column lanes (a power of two >= d) times RA_THREADS / W row lanes; the row lanes of a column
// are added in lane order.
__global__ void __launch_bounds__(RA_THREADS)
regadj_colsum_kernel(RaGroup g, int d, int64_t N, int64_t rows, int W, double* __restrict__ psum,
                     int64_t* __restrict__ pcount) {
    __shared__ double part[RA_THREADS];
    __shared__ int64_t npart[RA_THREADS];
    const int c = threadIdx.x % W, r = threadIdx.x / W, R = RA_THREADS / W;
    const int64_t i0 = int64_t(blockIdx.x) * rows;
    const int64_t i1 = i0 + rows < N ? i0 + rows : N;
    double s = 0.0;
    int64_t n = 0;
    for (int64_t i = i0 + r; i < i1; i += R) {
        if (!ra_member(g, i)) continue;
        ++n;
        if (c < d) s += ra_value(g, i, c);
    }
    part[threadIdx.x] = s;
    npart[threadIdx.x] = n;
    __syncthreads();
    if (r == 0 && c < d) {
        double t = part[c];
        for (int rr = 1; rr < R; ++rr) t += part[rr * W + c];
        psum[int64_t(blockIdx.x) * d + c] = t;
    }
    if (threadIdx.x == 0) {
        int64_t t = 0;
        for (int rr = 0; rr < R; ++rr) t += npart[rr * W];
        pcount[blockIdx.x] = t;
    }
}

// mom[0] = n_g, mom[1 + j] = mean of column j: left folds over the chunks
__global__ void __launch_bounds__(RA_THREADS)
regadj_mean_kernel(const double* __restrict__ psum, const int64_t* __restrict__ pcount,
                   int64_t n_chunks, int d, double* __restrict__ mom) {
    int64_t n = 0;
    for (int64_t c = 0; c < n_chunks; ++c) n += pcount[c];
    for (int j = threadIdx.x; j < d; j += RA_THREADS) {
        double t = 0.0;
        for (int64_t c = 0; c < n_chunks; ++c) t += psum[c * d + j];
        mom[1 + j] = t / double(n);
    }
    if (threadIdx.x == 0) mom[0] = double(n);
}

// lower tile index -> (ti, tj), tile = ti (ti + 1) / 2 + tj, tj <= ti
__device__ __forceinline__ void ra_lower_tile(int tile, int& ti, int& tj) {
    ti = 0;
    while ((ti + 1) * (ti + 2) / 2 <= tile) ++ti;
    tj = tile - ti * (ti + 1) / 2;
}

// P[(chunk * tiles + tile) * 64 * 64 + a * 64 + b] = sum over the chunk's group rows of
// (x_{r0 + a} - m)(x_{c0 + b} - m), from zero, rows in order.  Thread (ty, tx) owns rows ty + 16 u
// and columns tx + 16 v, u, v < 4, of the tile.
__global__ void __launch_bounds__(RA_THREADS)
regadj_cross_kernel(RaGroup g, int d, int64_t N, int64_t rows, int tiles,
                    const double* __restrict__ mom, double* __restrict__ P) {
    __shared__ double A[RA_SLAB][RA_TILE + 1];
    __shared__ double B[RA_SLAB][RA_TILE + 1];
    __shared__ double mean[RA_D_MAX];
    __shared__ bool member[RA_SLAB];
    const int tile = int(blockIdx.x % tiles);
    const int64_t chunk = blockIdx.x / tiles;
    int ti, tj;
    ra_lower_tile(tile, ti, tj);
    const int r0 = ti * RA_TILE, c0 = tj * RA_TILE;
    const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
    for (int j = threadIdx.x; j < d; j += RA_THREADS) mean[j] = mom[1 + j];
    const int64_t i0 = chunk * rows;
    const int64_t i1 = i0 + rows < N ? i0 + rows : N;
    double acc[4][4];
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) acc[u][v] = 0.0;
    for (int64_t rb = i0; rb < i1; rb += RA_SLAB) {
        if (threadIdx.x < RA_SLAB) {
            const int64_t i = rb + threadIdx.x;
            member[threadIdx.x] = i < i1 && ra_member(g, i);
        }
        __syncthreads();
        for (int e = threadIdx.x; e < RA_SLAB * RA_TILE; e += RA_THREADS) {
            const int ii = e / RA_TILE, cc = e % RA_TILE;
            const int64_t i = rb + ii;
            const int ja = r0 + cc, jb = c0 + cc;
            const bool m = member[ii];
            A[ii][cc] = (m && ja < d) ? ra_value(g, i, ja) - mean[ja] : 0.0;
            B[ii][cc] = (m && jb < d) ? ra_value(g, i, jb) - mean[jb] : 0.0;
        }
        __syncthreads();
#pragma unroll 4
        for (int ii = 0; ii < RA_SLAB; ++ii) {
            double a[4], b[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) a[u] = A[ii][ty + 16 * u];
#pragma unroll
            for (int v = 0; v < 4; ++v) b[v] = B[ii][tx + 16 * v];
#pragma unroll
            for (int u = 0; u < 4; ++u)
#pragma unroll
                for (int v = 0; v < 4; ++v) acc[u][v] = fma(a[u], b[v], acc[u][v]);
        }
        __syncthreads();
    }
    double* out = P + (chunk * tiles + tile) * int64_t(RA_TILE * RA_TILE);
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) out[(ty + 16 * u) * RA_TILE + tx + 16 * v] = acc[u][v];
}

// mom[1 + d + r * d + c] = mom[1 + d + c * d + r] = left fold over the chunks of P at (r, c), r >= c
__global__ void __launch_bounds__(RA_THREADS)
regadj_cross_reduce_kernel(const double* __restrict__ P, int64_t n_chunks, int tiles, int d,
                           double* __restrict__ mom) {
    const int64_t lower = int64_t(d) * (d + 1) / 2;
    for (int64_t e = int64_t(blockIdx.x) * RA_THREADS + threadIdx.x; e < lower;
         e += int64_t(gridDim.x) * RA_THREADS) {
        int r = int((sqrt(8.0 * double(e) + 1.0) - 1.0) / 2.0);
        while (int64_t(r) * (r + 1) / 2 > e) --r;
        while (int64_t(r + 1) * (r + 2) / 2 <= e) ++r;
        const int c = int(e - int64_t(r) * (r + 1) / 2);
        const int ti = r / RA_TILE, tj = c / RA_TILE;
        const int64_t off = int64_t(ti * (ti + 1) / 2 + tj) * RA_TILE * RA_TILE +
                            (r % RA_TILE) * RA_TILE + c % RA_TILE;
        double t = 0.0;
        for (int64_t k = 0; k < n_chunks; ++k) t += P[k * tiles * RA_TILE * RA_TILE + off];
        double* M = mom + 1 + d;
        M[int64_t(r) * d + c] = t;
        M[int64_t(c) * d + r] = t;
    }
}

// ccount[b] = the group's rows among rows [b RA_ADJ_ROWS, (b + 1) RA_ADJ_ROWS)
__global__ void __launch_bounds__(RA_THREADS)
regadj_count_kernel(RaGroup g, int64_t N, int64_t* __restrict__ ccount) {
    const int64_t i0 = int64_t(blockIdx.x) * RA_ADJ_ROWS;
    int64_t n = 0;
    for (int s = 0; s < RA_ADJ_ROWS; s += RA_THREADS) {
        const int64_t i = i0 + s + threadIdx.x;
        n += __syncthreads_count(i < N && ra_member(g, i));
    }
    if (threadIdx.x == 0) ccount[blockIdx.x] = n;
}

// the exclusive prefix sum of ccount[0 .. nb - 1], in place, by one CTA of 1024 threads
__global__ void __launch_bounds__(1024)
regadj_scan_kernel(int64_t* __restrict__ ccount, int64_t nb) {
    __shared__ int64_t seg[1024];
    const int64_t per = (nb + 1023) / 1024;
    const int64_t b0 = threadIdx.x * per;
    const int64_t b1 = b0 + per < nb ? b0 + per : nb;
    int64_t s = 0;
    for (int64_t b = b0; b < b1; ++b) s += ccount[b];
    seg[threadIdx.x] = s;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
        const int64_t v = threadIdx.x >= o ? seg[threadIdx.x - o] : 0;
        __syncthreads();
        seg[threadIdx.x] += v;
        __syncthreads();
    }
    int64_t run = seg[threadIdx.x] - s;
    for (int64_t b = b0; b < b1; ++b) {
        const int64_t c = ccount[b];
        ccount[b] = run;
        run += c;
    }
}

// out[k * ld_out + pos(i)] = T[i, cols[k]] - sum_j (S[i, j] - o_j) coef[j * pg + k] for the group's
// rows i of this CTA; pos(i) = i when dense, otherwise first[blockIdx.x] plus the rank of i among
// the CTA's group rows
__global__ void __launch_bounds__(RA_THREADS)
regadj_adjust_kernel(RaGroup g, int64_t N, int dense, const int64_t* __restrict__ first,
                     const double* __restrict__ coef, double* __restrict__ out, int64_t ld_out) {
    __shared__ int warp_n[RA_THREADS / 32];
    const int lane = threadIdx.x % 32, warp = threadIdx.x / 32;
    const int64_t i0 = int64_t(blockIdx.x) * RA_ADJ_ROWS;
    int64_t base = dense ? 0 : first[blockIdx.x];
    for (int s = 0; s < RA_ADJ_ROWS; s += RA_THREADS) {
        const int64_t i = i0 + s + threadIdx.x;
        const bool m = i < N && ra_member(g, i);
        int64_t pos = i;
        if (!dense) {
            const unsigned bal = __ballot_sync(0xffffffffu, m);
            if (lane == 0) warp_n[warp] = __popc(bal);
            __syncthreads();
            int before = 0, total = 0;
            for (int w = 0; w < RA_THREADS / 32; ++w) {
                before += w < warp ? warp_n[w] : 0;
                total += warp_n[w];
            }
            pos = base + before + __popc(bal & ((1u << lane) - 1u));
            base += total;
            __syncthreads();
        }
        if (!m) continue;
        const double* row = g.S + i * g.ldS;
        const double* t = g.T + i * g.ldT;
        for (int k0 = 0; k0 < g.pg; k0 += 4) {
            double acc[4] = {0.0, 0.0, 0.0, 0.0};
            const int kn = g.pg - k0 < 4 ? g.pg - k0 : 4;
            for (int j = 0; j < g.q; ++j) {
                const double x = row[j] - g.o[j];
                const double* cj = coef + int64_t(j) * g.pg + k0;
#pragma unroll
                for (int kk = 0; kk < 4; ++kk)
                    if (kk < kn) acc[kk] = fma(x, __ldg(cj + kk), acc[kk]);
            }
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
                if (kk < kn) out[int64_t(k0 + kk) * ld_out + pos] = t[g.cols[k0 + kk]] - acc[kk];
        }
    }
}

static size_t ra_align(size_t bytes) { return (bytes + 255) / 256 * 256; }

// the shared argument checks of the group entry points; cols_host is copied to `cols`
static int ra_group_args(const double* S, int64_t ldS, int64_t N, int64_t q, const double* obs,
                         const double* T, int64_t ldT, int64_t p, const uint8_t* flags,
                         const int32_t* cols_host, int64_t pg, int64_t sel, const char* who) {
    ELFI_REQUIRE(S && obs && T && flags && cols_host, "%s: NULL argument", who);
    ELFI_REQUIRE(q >= 1 && p >= 1 && q + p <= RA_D_MAX && N >= 1 && N <= ELFI_B200_REGADJ_N_MAX &&
                     ldS >= q && ldT >= p,
                 "%s: bad shape (q, p >= 1, q + p <= %d, 1 <= N < 2^31, ldS >= q, ldT >= p; "
                 "N=%lld q=%lld p=%lld ldS=%lld ldT=%lld)", who, RA_D_MAX, (long long)N,
                 (long long)q, (long long)p, (long long)ldS, (long long)ldT);
    ELFI_REQUIRE(pg >= 1 && pg <= p && sel >= -1 && sel < p,
                 "%s: 1 <= pg <= p and -1 <= sel < p (pg=%lld sel=%lld p=%lld)", who, (long long)pg,
                 (long long)sel, (long long)p);
    for (int64_t k = 0; k < pg; ++k)
        ELFI_REQUIRE(cols_host[k] >= 0 && cols_host[k] < p,
                     "%s: parameter column %lld is %d, outside [0, %lld)", who, (long long)k,
                     int(cols_host[k]), (long long)p);
    return ELFI_B200_OK;
}

}  // namespace elfi

extern "C" {

int elfi_b200_regadj_mask_f64(elfi_b200_ctx* ctx, const double* S, int64_t ldS, int64_t N,
                              int64_t q, const double* obs, const double* T, int64_t ldT, int64_t p,
                              uint8_t* flags, int64_t* counts, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && S && obs && T && flags && counts, "regadj_mask: NULL argument");
    ELFI_REQUIRE(q >= 1 && p >= 1 && q + p <= RA_D_MAX && N >= 1 && N <= ELFI_B200_REGADJ_N_MAX &&
                     ldS >= q && ldT >= p,
                 "regadj_mask: bad shape (q, p >= 1, q + p <= %d, 1 <= N < 2^31, ldS >= q, "
                 "ldT >= p; N=%lld q=%lld p=%lld ldS=%lld ldT=%lld)", RA_D_MAX, (long long)N,
                 (long long)q, (long long)p, (long long)ldS, (long long)ldT);
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        ELFI_CUDA_OK(cudaMemsetAsync(counts, 0, size_t(p + 1) * 8, stream));
        regadj_mask_kernel<<<capped_grid(ctx, N, RA_THREADS, 8), RA_THREADS, 0, stream>>>(
            S, ldS, N, int(q), obs, T, ldT, int(p), flags,
            reinterpret_cast<unsigned long long*>(counts));
        return ELFI_B200_OK;
    });
}

int elfi_b200_regadj_moments_f64(elfi_b200_ctx* ctx, const double* S, int64_t ldS, int64_t N,
                                 int64_t q, const double* obs, const double* T, int64_t ldT,
                                 int64_t p, const uint8_t* flags, const int32_t* cols_host,
                                 int64_t pg, int64_t sel, double* mom, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && mom, "regadj_moments: NULL argument");
    const int rc = ra_group_args(S, ldS, N, q, obs, T, ldT, p, flags, cols_host, pg, sel,
                                 "regadj_moments");
    if (rc != ELFI_B200_OK) return rc;
    const int d = int(q + pg);
    const RaChunks ch = ra_chunks(N, d);
    const size_t b_cols = ra_align(size_t(pg) * 4);
    const size_t b_psum = ra_align(size_t(ch.n) * d * 8);
    const size_t b_pcount = ra_align(size_t(ch.n) * 8);
    const size_t b_P = size_t(ch.n) * ch.tiles * RA_TILE * RA_TILE * 8;
    uint8_t* base = static_cast<uint8_t*>(ctx_scratch(ctx, b_cols + b_psum + b_pcount + b_P));
    if (!base) return ELFI_B200_ERR_NOMEM;
    int32_t* cols = reinterpret_cast<int32_t*>(base);
    double* psum = reinterpret_cast<double*>(base + b_cols);
    int64_t* pcount = reinterpret_cast<int64_t*>(base + b_cols + b_psum);
    double* P = reinterpret_cast<double*>(base + b_cols + b_psum + b_pcount);
    const RaGroup g{S, ldS, obs, T, ldT, flags, cols, int(q), int(pg), int(sel)};
    int W = 1;
    while (W < d) W *= 2;
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        ELFI_CUDA_OK(cudaMemcpyAsync(cols, cols_host, size_t(pg) * 4, cudaMemcpyHostToDevice,
                                     stream));
        regadj_colsum_kernel<<<unsigned(ch.n), RA_THREADS, 0, stream>>>(g, d, N, ch.rows, W, psum,
                                                                        pcount);
        regadj_mean_kernel<<<1, RA_THREADS, 0, stream>>>(psum, pcount, ch.n, d, mom);
        regadj_cross_kernel<<<unsigned(ch.n * ch.tiles), RA_THREADS, 0, stream>>>(
            g, d, N, ch.rows, ch.tiles, mom, P);
        const int64_t lower = int64_t(d) * (d + 1) / 2;
        regadj_cross_reduce_kernel<<<unsigned((lower + RA_THREADS - 1) / RA_THREADS), RA_THREADS,
                                     0, stream>>>(P, ch.n, ch.tiles, d, mom);
        return ELFI_B200_OK;
    });
}

int elfi_b200_regadj_adjust_f64(elfi_b200_ctx* ctx, const double* S, int64_t ldS, int64_t N,
                                int64_t q, const double* obs, const double* T, int64_t ldT,
                                int64_t p, const uint8_t* flags, const int32_t* cols_host,
                                int64_t pg, int64_t sel, int32_t dense, const double* coef,
                                double* out, int64_t ld_out, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && coef && out, "regadj_adjust: NULL argument");
    const int rc = ra_group_args(S, ldS, N, q, obs, T, ldT, p, flags, cols_host, pg, sel,
                                 "regadj_adjust");
    if (rc != ELFI_B200_OK) return rc;
    ELFI_REQUIRE(dense == 0 || dense == 1, "regadj_adjust: dense must be 0 or 1, got %d",
                 int(dense));
    ELFI_REQUIRE(ld_out >= (dense ? N : 1), "regadj_adjust: ld_out=%lld is below %lld",
                 (long long)ld_out, (long long)(dense ? N : 1));
    const int64_t nb = (N + RA_ADJ_ROWS - 1) / RA_ADJ_ROWS;
    const size_t b_cols = ra_align(size_t(pg) * 4);
    uint8_t* base = static_cast<uint8_t*>(ctx_scratch(ctx, b_cols + size_t(nb) * 8));
    if (!base) return ELFI_B200_ERR_NOMEM;
    int32_t* cols = reinterpret_cast<int32_t*>(base);
    int64_t* first = reinterpret_cast<int64_t*>(base + b_cols);
    const RaGroup g{S, ldS, obs, T, ldT, flags, cols, int(q), int(pg), int(sel)};
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        ELFI_CUDA_OK(cudaMemcpyAsync(cols, cols_host, size_t(pg) * 4, cudaMemcpyHostToDevice,
                                     stream));
        if (!dense) {
            regadj_count_kernel<<<unsigned(nb), RA_THREADS, 0, stream>>>(g, N, first);
            regadj_scan_kernel<<<1, 1024, 0, stream>>>(first, nb);
        }
        regadj_adjust_kernel<<<unsigned(nb), RA_THREADS, 0, stream>>>(g, N, int(dense), first, coef,
                                                                      out, ld_out);
        return ELFI_B200_OK;
    });
}

}  // extern "C"
