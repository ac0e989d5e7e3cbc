// synlik.cu -- the Gaussian synthetic log-likelihood of Bayesian synthetic likelihood (BSL;
// elfi/methods/bsl/pdf_methods.py: gaussian_syn_likelihood with Warton shrinkage and whitening,
// gaussian_syn_likelihood_ghurye_olkin) for G groups of n simulated summary rows.
//
// Launches, in stream order:
//   1. synlik_mean_kernel: the column means mu (G x d), one CTA per (group, 32 columns).
//   2. synlik_cross_kernel: the centred cross-products sum_i (x_i - mu)(x_i - mu)^T, lower 32 x 32
//      tiles only.  Rows are taken in chunks of SL_CHUNK; each chunk's products are summed from
//      zero, and the chunk sums are added left to right.  When G alone does not fill the GPU each
//      chunk is its own CTA and writes its sum to scratch ("split"); otherwise one CTA walks all
//      chunks of its tile.  Both give the same bits, since the left fold over the chunk sums is the
//      same, so a group's result does not depend on G, K or the other groups.  No atomics.
//   3. synlik_reduce_kernel (split, or whitening): the left fold over the chunk sums, times
//      1 / (n - 1), mirrored to a full symmetric Sigma.
//   4. whitening: W Sigma W^T as two batched NT products through scratch (synlik_gemm_nt_kernel).
//   5. synlik_factor_kernel: one CTA per (group, penalty).  It shrinks Sigma into shared memory,
//      appends the right-hand side b = y_g - mu (or W (y_g - mu)) as row d, where y_g is the
//      group's observation (one row shared by every group, or one row per group), and runs a
//      right-looking Cholesky over the d + 1 rows: row d then holds z = L^{-1} b, so one
//      factorisation gives
//      log det Sigma = 2 sum log L_jj and m = |z|^2.
#include <cfloat>
#include <cmath>

#include "common.cuh"

namespace elfi {

constexpr int SL_D_MAX = ELFI_B200_SYNLIK_D_MAX;
constexpr int SL_TILE = 32;
constexpr int SL_CHUNK = 256;          // rows of one chunk sum: fixes the summation order
constexpr int SL_THREADS = 256;
constexpr double SL_WARTON_EPS = 1e-5;
// most bytes of chunk sums kept in scratch by the split form; larger problems walk their chunks
// inside one CTA
constexpr size_t SL_SPLIT_BYTES = size_t(256) << 20;

// mu[g * d + j] = mean of column j of group g; 8 row lanes per column, added in lane order
__global__ void __launch_bounds__(SL_THREADS)
synlik_mean_kernel(const double* __restrict__ S, int64_t ld_row, int64_t ld_group, int n, int d,
                   int col_tiles, double* __restrict__ mu) {
    __shared__ double part[SL_THREADS / SL_TILE][SL_TILE];
    const int64_t g = blockIdx.x / col_tiles;
    const int tx = threadIdx.x % SL_TILE, ty = threadIdx.x / SL_TILE;
    const int j = int(blockIdx.x % col_tiles) * SL_TILE + tx;
    double s = 0.0;
    if (j < d) {
        const double* col = S + g * ld_group + j;
        for (int i = ty; i < n; i += SL_THREADS / SL_TILE) s += col[int64_t(i) * ld_row];
    }
    part[ty][tx] = s;
    __syncthreads();
    if (ty == 0 && j < d) {
        double t = part[0][tx];
        for (int q = 1; q < SL_THREADS / SL_TILE; ++q) t += part[q][tx];
        mu[g * d + j] = t / n;
    }
}

// lower tile index -> (ti, tj), tile = ti (ti + 1) / 2 + tj, tj <= ti
__device__ __forceinline__ void lower_tile(int tile, int& ti, int& tj) {
    ti = 0;
    while ((ti + 1) * (ti + 2) / 2 <= tile) ++ti;
    tj = tile - ti * (ti + 1) / 2;
}

// P[(g * n_parts + part) * d * d + r * d + c] for (r, c) in the lower tiles: the left fold over
// the chunk sums of chunks [part * cpc, (part + 1) * cpc).  Thread (ty, tx) owns rows ty + 8 q,
// q < 4, of column tx of the tile.
__global__ void __launch_bounds__(SL_THREADS)
synlik_cross_kernel(const double* __restrict__ S, int64_t ld_row, int64_t ld_group, int n, int d,
                    const double* __restrict__ mu, int n_tiles, int n_parts, int cpc,
                    double* __restrict__ P) {
    __shared__ double A[SL_TILE][SL_TILE + 1];
    __shared__ double Bt[SL_TILE][SL_TILE + 1];
    int64_t bid = blockIdx.x;
    const int part = int(bid % n_parts);
    bid /= n_parts;
    const int tile = int(bid % n_tiles);
    const int64_t g = bid / n_tiles;
    int ti, tj;
    lower_tile(tile, ti, tj);
    const int r0 = ti * SL_TILE, c0 = tj * SL_TILE;
    const int tx = threadIdx.x % SL_TILE, ty = threadIdx.x / SL_TILE;
    const double* Sg = S + g * ld_group;
    const double* mug = mu + g * d;
    const int n_chunks = (n + SL_CHUNK - 1) / SL_CHUNK;
    const int ch_end = min(n_chunks, (part + 1) * cpc);
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    for (int ch = part * cpc; ch < ch_end; ++ch) {
        double p[4] = {0.0, 0.0, 0.0, 0.0};
        for (int rb = ch * SL_CHUNK; rb < (ch + 1) * SL_CHUNK && rb < n; rb += SL_TILE) {
            for (int e = threadIdx.x; e < SL_TILE * SL_TILE; e += SL_THREADS) {
                const int ii = e / SL_TILE, cc = e % SL_TILE;
                const int i = rb + ii;
                const int ja = r0 + cc, jb = c0 + cc;
                const double* row = Sg + int64_t(i) * ld_row;
                A[ii][cc] = (i < n && ja < d) ? row[ja] - mug[ja] : 0.0;
                Bt[ii][cc] = (i < n && jb < d) ? row[jb] - mug[jb] : 0.0;
            }
            __syncthreads();
#pragma unroll 8
            for (int ii = 0; ii < SL_TILE; ++ii) {
                const double b = Bt[ii][tx];
#pragma unroll
                for (int q = 0; q < 4; ++q) p[q] = fma(A[ii][ty + 8 * q], b, p[q]);
            }
            __syncthreads();
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[q] += p[q];
    }
    double* Pg = P + (g * n_parts + part) * int64_t(d) * d;
    const int c = c0 + tx;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int r = r0 + ty + 8 * q;
        if (r < d && c < d) Pg[int64_t(r) * d + c] = acc[q];
    }
}

// R[g * d * d + i * d + j] = scale * (left fold over the parts of P at (max(i, j), min(i, j)))
__global__ void __launch_bounds__(SL_THREADS)
synlik_reduce_kernel(const double* __restrict__ P, int64_t G, int d, int n_parts, double scale,
                     double* __restrict__ R) {
    const int64_t dd = int64_t(d) * d;
    const int64_t e = int64_t(blockIdx.x) * SL_THREADS + threadIdx.x;
    if (e >= G * dd) return;
    const int64_t g = e / dd;
    const int i = int((e % dd) / d), j = int(e % d);
    const int64_t at = int64_t(max(i, j)) * d + min(i, j);
    double acc = 0.0;
    for (int p = 0; p < n_parts; ++p) acc += P[(g * n_parts + p) * dd + at];
    R[e] = acc * scale;
}

// C[g] = A[g] B[g]^T for d x d row-major matrices at group strides sA, sB, sC (0: shared)
__global__ void __launch_bounds__(SL_THREADS)
synlik_gemm_nt_kernel(const double* __restrict__ A, int64_t sA, const double* __restrict__ B,
                      int64_t sB, double* __restrict__ C, int64_t sC, int d, int tiles) {
    __shared__ double As[SL_TILE][SL_TILE + 1];
    __shared__ double Bs[SL_TILE][SL_TILE + 1];
    const int64_t g = blockIdx.x / (tiles * tiles);
    const int t = int(blockIdx.x % (tiles * tiles));
    const int r0 = (t / tiles) * SL_TILE, c0 = (t % tiles) * SL_TILE;
    const int tx = threadIdx.x % SL_TILE, ty = threadIdx.x / SL_TILE;
    const double* Ag = A + g * sA;
    const double* Bg = B + g * sB;
    double p[4] = {0.0, 0.0, 0.0, 0.0};
    for (int k0 = 0; k0 < d; k0 += SL_TILE) {
        for (int e = threadIdx.x; e < SL_TILE * SL_TILE; e += SL_THREADS) {
            const int rr = e / SL_TILE, kk = e % SL_TILE;
            const int k = k0 + kk;
            As[rr][kk] = (r0 + rr < d && k < d) ? Ag[int64_t(r0 + rr) * d + k] : 0.0;
            Bs[rr][kk] = (c0 + rr < d && k < d) ? Bg[int64_t(c0 + rr) * d + k] : 0.0;
        }
        __syncthreads();
#pragma unroll 8
        for (int kk = 0; kk < SL_TILE; ++kk) {
            const double b = Bs[tx][kk];
#pragma unroll
            for (int q = 0; q < 4; ++q) p[q] = fma(As[ty + 8 * q][kk], b, p[q]);
        }
        __syncthreads();
    }
    double* Cg = C + g * sC;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int r = r0 + ty + 8 * q, c = c0 + tx;
        if (r < d && c < d) Cg[int64_t(r) * d + c] = p[q];
    }
}

// sum over j < d of f(j), in an order fixed by d alone (lane-strided, then a shuffle tree);
// warp 0 only, the result in lane 0
template <class F>
__device__ __forceinline__ double warp_sum(int d, F&& f) {
    const int lane = threadIdx.x % 32;
    double s = 0.0;
    for (int j = lane; j < d; j += 32) s += f(j);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    return s;
}

// shared-memory doubles of the factor kernel at dimension d
__host__ __device__ constexpr int64_t synlik_factor_doubles(int d) {
    return int64_t(d + 1) * (d + 1) + (d + 1) + d;
}

// loglik[g * max(K, 1) + k] for group g and penalty k (lambda = 0 when K = 0).  Sig holds the
// group's covariance at Sig[g * d * d + i * d + j], i >= j read, times scale; the group's
// observation is y + g * ld_y (ld_y = 0: one row for every group).
__global__ void __launch_bounds__(512)
synlik_factor_kernel(const double* __restrict__ Sig, double scale, const double* __restrict__ mu,
                     const double* __restrict__ y, int64_t ld_y, const double* __restrict__ W,
                     const double* __restrict__ pen, int K, int d, int estimator, double n,
                     double c_unbiased, double* __restrict__ loglik) {
    extern __shared__ double sm[];
    const int ld = d + 1;
    double* L = sm;                      // rows 0 .. d - 1: Sigma_lambda -> L; row d: b -> z
    double* col = L + int64_t(d + 1) * ld;   // column j of L below the diagonal, and z_j
    double* dg = col + (d + 1);              // L_jj
    __shared__ double maxdiag;
    const int64_t g = blockIdx.x;
    const int k = blockIdx.y;
    const int tid = threadIdx.x, nthr = blockDim.x;
    const int lane = tid % 32, warp = tid / 32, nwarps = nthr / 32;
    const double lam = K ? pen[k] : 0.0;
    const double* Sg = Sig + g * int64_t(d) * d;
    const double* mug = mu + g * d;
    const double* yg = y + g * ld_y;
    double* out = loglik + g * (K ? K : 1) + k;

    // a non-finite input makes its column sum, so its mean, non-finite
    bool bad = false;
    for (int j = tid; j < d; j += nthr) bad |= !isfinite(mug[j]);
    if (__syncthreads_or(bad)) {
        if (tid == 0) *out = -INFINITY;
        return;
    }
    for (int i = warp; i < d; i += nwarps) {
        for (int j = lane; j <= i; j += 32) {
            double v = Sg[int64_t(i) * d + j] * scale;
            if (K) v = (i == j) ? (1.0 - lam) * v + lam * (v + SL_WARTON_EPS) : (1.0 - lam) * v;
            L[i * ld + j] = v;
        }
    }
    for (int j = tid; j < d; j += nthr) col[j] = yg[j] - mug[j];
    __syncthreads();
    for (int i = tid; i < d; i += nthr) {
        double b = col[i];
        if (W) {
            b = 0.0;
            for (int j = 0; j < d; ++j) b = fma(W[int64_t(i) * d + j], col[j], b);
        }
        L[d * ld + i] = b;
    }
    if (warp == 0) {
        double mx = 0.0;
        for (int j = lane; j < d; j += 32) mx = fmax(mx, L[j * ld + j]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        if (lane == 0) maxdiag = mx;
    }
    __syncthreads();
    const double thr = 1e6 * DBL_EPSILON * maxdiag;

    for (int j = 0; j < d; ++j) {
        const double piv = L[j * ld + j];          // read by every thread: the exit is uniform
        if (!(piv > thr) || !isfinite(piv)) {
            if (tid == 0) *out = -INFINITY;
            return;
        }
        const double ljj = sqrt(piv);
        for (int i = j + 1 + tid; i <= d; i += nthr) {
            const double v = L[i * ld + j] / ljj;
            L[i * ld + j] = v;
            col[i] = v;
        }
        if (tid == 0) dg[j] = ljj;
        __syncthreads();
        for (int i = j + 1 + warp; i <= d; i += nwarps) {
            const double lij = col[i];
            const int kend = i < d ? i : d - 1;
            for (int c = j + 1 + lane; c <= kend; c += 32) L[i * ld + c] -= lij * col[c];
        }
        __syncthreads();
    }
    if (warp != 0) return;
    const double* z = L + d * ld;
    const double logdet = 2.0 * warp_sum(d, [&](int j) { return log(dg[j]); });
    const double m = warp_sum(d, [&](int j) { return z[j] * z[j]; });
    if (lane != 0) return;
    double ll;
    if (estimator == 0) {
        ll = -0.5 * (d * log(2.0 * M_PI) + logdet + m);
    } else {
        const double l1 = log(n - 1.0);
        const double logdet_psi = d * l1 + logdet + log(fabs(1.0 - n * m / ((n - 1.0) * (n - 1.0))));
        ll = c_unbiased - 0.5 * (n - d - 2.0) * (l1 + logdet) + 0.5 * (n - d - 3.0) * logdet_psi;
    }
    *out = ll;
}

// log c(k, nu) of Ghurye and Olkin (1969)
static double log_c(int64_t k, double nu) {
    double s = -double(k) * nu / 2.0 * std::log(2.0) - double(k) * (k - 1) / 4.0 * std::log(M_PI);
    for (int64_t i = 0; i < k; ++i) s -= std::lgamma(0.5 * (nu - double(i)));
    return s;
}

static size_t align256(size_t bytes) { return (bytes + 255) / 256 * 256; }

// both entry points: group g's observation is y + g * ld_y (ld_y = 0: one row for every group)
static int synlik_launch(elfi_b200_ctx* ctx, const double* S, int64_t ld_row, int64_t ld_group,
                         int64_t G, int64_t n, int64_t d, const double* y, int64_t ld_y,
                         const double* W, int32_t estimator, const double* penalties_host,
                         int64_t K, double* loglik, void* stream_) {
    ELFI_REQUIRE(ctx && (G == 0 || (S && y && loglik)), "synlik: NULL argument");
    ELFI_REQUIRE(ld_y == 0 || ld_y >= d,
                 "synlik: the observation stride must be 0 or at least d (ld_y=%lld d=%lld)",
                 (long long)ld_y, (long long)d);
    ELFI_REQUIRE(d >= 1 && d <= SL_D_MAX && n >= 2 && n < (int64_t(1) << 31) && G >= 0 &&
                     G <= (int64_t(1) << 22) && ld_row >= d && ld_group >= 0,
                 "synlik: bad shape (1 <= d <= %d, 2 <= n < 2^31, G <= 2^22, ld_row >= d, "
                 "ld_group >= 0; "
                 "G=%lld n=%lld d=%lld ld_row=%lld ld_group=%lld)", SL_D_MAX, (long long)G,
                 (long long)n, (long long)d, (long long)ld_row, (long long)ld_group);
    ELFI_REQUIRE(estimator == 0 || estimator == 1,
                 "synlik: estimator must be 0 (standard) or 1 (unbiased), got %d", int(estimator));
    ELFI_REQUIRE(estimator == 0 || (W == nullptr && K == 0),
                 "synlik: whitening and penalties apply to the standard estimator only");
    ELFI_REQUIRE(K >= 0 && K <= 65535 && (K == 0 || penalties_host),
                 "synlik: 0 <= K <= 65535 penalties, given on the host (K=%lld)", (long long)K);
    for (int64_t k = 0; k < K; ++k)
        ELFI_REQUIRE(penalties_host[k] >= 0.0 && penalties_host[k] <= 1.0,
                     "synlik: Warton penalty %lld is %g, outside [0, 1]", (long long)k,
                     penalties_host[k]);
    if (G == 0) return ELFI_B200_OK;

    const int di = int(d), ni = int(n);
    const int col_tiles = (di + SL_TILE - 1) / SL_TILE;
    const int n_tiles = col_tiles * (col_tiles + 1) / 2;
    const int n_chunks = (ni + SL_CHUNK - 1) / SL_CHUNK;
    const size_t dd = size_t(d) * d;
    const bool split = n_chunks > 1 && G * n_tiles < 2 * int64_t(ctx->sm_count) &&
                       size_t(G) * n_chunks * dd * 8 <= SL_SPLIT_BYTES;
    const int n_parts = split ? n_chunks : 1;
    const bool reduce = split || W;
    const size_t b_mu = align256(size_t(G) * d * 8);
    const size_t b_P = align256(size_t(G) * n_parts * dd * 8);
    const size_t b_R = reduce ? align256(size_t(G) * dd * 8) : 0;
    const size_t b_W = W ? 2 * align256(size_t(G) * dd * 8) : 0;
    const size_t b_pen = align256(size_t(K) * 8);
    uint8_t* base = static_cast<uint8_t*>(ctx_scratch(ctx, b_mu + b_P + b_R + b_W + b_pen));
    if (!base) return ELFI_B200_ERR_NOMEM;
    double* mu = reinterpret_cast<double*>(base);
    double* P = reinterpret_cast<double*>(base + b_mu);
    double* R = reinterpret_cast<double*>(base + b_mu + b_P);
    double* T = reinterpret_cast<double*>(base + b_mu + b_P + b_R);
    double* Sw = T + G * dd;
    double* pen = reinterpret_cast<double*>(base + b_mu + b_P + b_R + b_W);
    const double c_unb = estimator == 1
        ? -0.5 * d * std::log(2.0 * M_PI) + log_c(d, double(n - 2)) - log_c(d, double(n - 1)) -
              0.5 * d * std::log(1.0 - 1.0 / double(n))
        : 0.0;
    const int factor_threads = di <= 64 ? 256 : 512;
    const size_t factor_smem = size_t(synlik_factor_doubles(di)) * 8;
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        if (K)
            ELFI_CUDA_OK(cudaMemcpyAsync(pen, penalties_host, size_t(K) * 8,
                                         cudaMemcpyHostToDevice, stream));
        synlik_mean_kernel<<<unsigned(G * col_tiles), SL_THREADS, 0, stream>>>(
            S, ld_row, ld_group, ni, di, col_tiles, mu);
        synlik_cross_kernel<<<unsigned(G * n_tiles * n_parts), SL_THREADS, 0, stream>>>(
            S, ld_row, ld_group, ni, di, mu, n_tiles, n_parts, split ? 1 : n_chunks, P);
        const double scale = 1.0 / double(n - 1);
        const double* sig = P;
        double sig_scale = scale;
        if (reduce) {
            synlik_reduce_kernel<<<unsigned((G * dd + SL_THREADS - 1) / SL_THREADS), SL_THREADS, 0,
                                   stream>>>(P, G, di, n_parts, scale, R);
            sig = R;
            sig_scale = 1.0;
        }
        if (W) {
            const unsigned blocks = unsigned(G * col_tiles * col_tiles);
            synlik_gemm_nt_kernel<<<blocks, SL_THREADS, 0, stream>>>(W, 0, R, int64_t(dd), T,
                                                                    int64_t(dd), di, col_tiles);
            synlik_gemm_nt_kernel<<<blocks, SL_THREADS, 0, stream>>>(T, int64_t(dd), W, 0, Sw,
                                                                    int64_t(dd), di, col_tiles);
            sig = Sw;
        }
        ELFI_CUDA_OK(cudaFuncSetAttribute(synlik_factor_kernel,
                                          cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          int(synlik_factor_doubles(SL_D_MAX) * 8)));
        synlik_factor_kernel<<<dim3(unsigned(G), unsigned(K ? K : 1)), factor_threads, factor_smem,
                               stream>>>(sig, sig_scale, mu, y, ld_y, W, pen, int(K), di,
                                         int(estimator), double(n), c_unb, loglik);
        return ELFI_B200_OK;
    });
}

}  // namespace elfi

extern "C" {

int elfi_b200_synlik_f64(elfi_b200_ctx* ctx, const double* S, int64_t ld_row, int64_t ld_group,
                         int64_t G, int64_t n, int64_t d, const double* y, const double* W,
                         int32_t estimator, const double* penalties_host, int64_t K,
                         double* loglik, void* stream) {
    return elfi::synlik_launch(ctx, S, ld_row, ld_group, G, n, d, y, 0, W, estimator,
                               penalties_host, K, loglik, stream);
}

int elfi_b200_synlik_obs_f64(elfi_b200_ctx* ctx, const double* S, int64_t ld_row,
                             int64_t ld_group, int64_t G, int64_t n, int64_t d, const double* Y,
                             int64_t ld_y, const double* W, int32_t estimator,
                             const double* penalties_host, int64_t K, double* loglik,
                             void* stream) {
    return elfi::synlik_launch(ctx, S, ld_row, ld_group, G, n, d, Y, ld_y, W, estimator,
                               penalties_host, K, loglik, stream);
}

}  // extern "C"
