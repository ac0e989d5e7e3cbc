// logreg.cu -- the ratio-estimation classifier of BOLFIRE (elfi/methods/classifier.py:
// LogisticRegression, i.e. sklearn's StandardScaler followed by liblinear's L1- or L2-penalised
// logistic regression with intercept_scaling = 1), fitted to the optimum on the device.
//
// elfi_b200_logreg_fit_f64 is one kernel launch with one CTA (LR_THREADS threads) per fit:
//   1. the labels are counted and the columns standardised (mean, ddof-0 variance, sklearn's
//      constant-column rule);
//   2. proximal Newton iterations (newGLMNET): one pass over the rows gives the loss, the
//      per-row gradient and curvature weights; a column pass gives the gradient g; the stopping
//      rule is tested; the lower 32 x 32 tiles of H = X~^T diag(h) X~ are accumulated row chunk by
//      row chunk through shared memory into a packed lower triangle; warp 0 runs coordinate
//      descent on the quadratic model (soft-thresholded for L1); a warp per row gives the step's
//      margins q = X~ delta; an Armijo line search on the precomputed margins picks the step.
//   3. the result block (header, mean_, scale_, coef_) is written by thread 0.
// Every reduction has an order fixed by (n, d) alone: strided per-thread partials, a shuffle tree,
// then the warps in order.  No atomics; repeated calls give the same bits.
// elfi_b200_logreg_predict_f64 is one thread per query row.
#include <cfloat>
#include <cmath>

#include "common.cuh"

namespace elfi {

constexpr int LR_D_MAX = ELFI_B200_LOGREG_D_MAX;
constexpr int LR_THREADS = 256;
constexpr int LR_WARPS = LR_THREADS / 32;
constexpr int LR_TILE = 32;
constexpr int LR_HEAD = ELFI_B200_LOGREG_HEAD;   // header doubles of the result block
constexpr int LR_MAX_SWEEPS = 1000;     // coordinate-descent sweeps per Newton step
constexpr int LR_MAX_HALVINGS = 40;     // line-search step halvings
constexpr double LR_ARMIJO = 0.01;      // sufficient-decrease fraction of the predicted decrease
constexpr double LR_TOL = 1e-10;        // stop when the min-norm subgradient <= LR_TOL * C * n
constexpr double LR_NU = 1e-12;         // added to diag(H) of the L1 model (newGLMNET's nu)

enum { LR_NOT_CONVERGED = 0, LR_CONVERGED = 1, LR_BAD_LABELS = -1, LR_NONFINITE = -2 };

static_assert(LR_THREADS == LR_WARPS * 32 && LR_THREADS / LR_TILE == LR_WARPS, "layout");

// shared-memory doubles of the fit kernel at dimension d (D = d + 1 with the intercept)
__host__ __device__ constexpr int64_t logreg_smem_doubles(int d) {
    return int64_t(d + 1) * (d + 2) / 2 + 2 * LR_TILE * (LR_TILE + 1) + 7 * int64_t(d + 1);
}

__device__ __forceinline__ int lr_packed(int r, int c) {   // (r, c) of the symmetric H, packed lower
    return r >= c ? r * (r + 1) / 2 + c : c * (c + 1) / 2 + r;
}

// sum of every thread's s in a fixed order (shuffle tree, then the warps in order); every thread
// gets the same value
__device__ __forceinline__ double lr_block_sum(double s, double* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    __syncthreads();
    if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = s;
    __syncthreads();
    double t = red[0];
#pragma unroll
    for (int q = 1; q < LR_WARPS; ++q) t += red[q];
    return t;
}

__device__ __forceinline__ double lr_block_max(double s, double* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s = fmax(s, __shfl_xor_sync(0xffffffffu, s, o));
    __syncthreads();
    if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = s;
    __syncthreads();
    double t = red[0];
#pragma unroll
    for (int q = 1; q < LR_WARPS; ++q) t = fmax(t, red[q]);
    return t;
}

// out[j] = sum_i wgt(i) val(i, j), j < ncols: row lane ty takes rows ty + 8 k in order, the eight
// row lanes are added in order
template <class Wf, class Vf>
__device__ __forceinline__ void lr_col_sums(int n, int ncols, Wf wgt, Vf val, double* out,
                                            double (*part)[LR_TILE]) {
    const int tx = threadIdx.x % LR_TILE, ty = threadIdx.x / LR_TILE;
    for (int c0 = 0; c0 < ncols; c0 += LR_TILE) {
        const int j = c0 + tx;
        double s = 0.0;
        if (j < ncols)
            for (int i = ty; i < n; i += LR_WARPS) s = fma(wgt(i), val(i, j), s);
        part[ty][tx] = s;
        __syncthreads();
        if (ty == 0 && j < ncols) {
            double t = part[0][tx];
#pragma unroll
            for (int q = 1; q < LR_WARPS; ++q) t += part[q][tx];
            out[j] = t;
        }
        __syncthreads();
    }
}

// log(1 + exp(-s)) without overflow
__device__ __forceinline__ double lr_loss(double s) {
    return log1p(exp(-fabs(s))) + fmax(-s, 0.0);
}

// the entry of the minimum-norm subgradient of F at coordinate j
__device__ __forceinline__ double lr_subgrad(double gj, double wj, bool l1) {
    if (!l1) return fabs(gj);
    if (wj > 0.0) return fabs(gj + 1.0);
    if (wj < 0.0) return fabs(gj - 1.0);
    return fmax(fabs(gj) - 1.0, 0.0);
}

__global__ void __launch_bounds__(LR_THREADS, 1)
logreg_fit_kernel(const double* __restrict__ X, int64_t ld, const double* __restrict__ y, int n,
                  int d, int penalty, double C, int max_iter, double* __restrict__ wx,
                  double* __restrict__ q, double* __restrict__ cg, double* __restrict__ ch,
                  double* __restrict__ out) {
    extern __shared__ double sm[];
    const int D = d + 1;
    const bool l1 = penalty == 0;
    double* H = sm;                                        // packed lower triangle of H
    double* A = H + D * (D + 1) / 2;                       // row tiles of X~ diag(h) and X~
    double* Bt = A + LR_TILE * (LR_TILE + 1);
    double* w = Bt + LR_TILE * (LR_TILE + 1);              // weights, intercept last
    double* g = w + D;                                     // gradient of the smooth part
    double* dl = g + D;                                    // Newton direction
    double* r = dl + D;                                    // gradient of the quadratic model
    double* mean = r + D;
    double* scale = mean + D;
    double* tmp = scale + D;
    __shared__ double red[LR_WARPS];
    __shared__ double part[LR_WARPS][LR_TILE];
    __shared__ double s_inner;
    const int tid = threadIdx.x, lane = tid % 32, warp = tid / 32;
    const double dn = double(n);

    auto xt = [&](int i, int j) -> double {                // standardised X with a trailing 1
        return j < d ? (X[int64_t(i) * ld + j] - mean[j]) / scale[j] : 1.0;
    };

    // ---- labels and standardisation -----------------------------------------------------------
    double npos = 0.0, nneg = 0.0, nbad = 0.0;
    for (int i = tid; i < n; i += LR_THREADS) {
        const double yi = y[i];
        npos += yi == 1.0;
        nneg += yi == -1.0;
        nbad += yi != 1.0 && yi != -1.0;
    }
    npos = lr_block_sum(npos, red);
    nneg = lr_block_sum(nneg, red);
    nbad = lr_block_sum(nbad, red);
    int status = (nbad > 0.0 || npos == 0.0 || nneg == 0.0) ? LR_BAD_LABELS : LR_NOT_CONVERGED;

    auto one = [](int) { return 1.0; };
    lr_col_sums(n, d, one, [&](int i, int j) { return X[int64_t(i) * ld + j]; }, tmp, part);
    for (int j = tid; j < d; j += LR_THREADS) mean[j] = tmp[j] / dn;
    __syncthreads();
    lr_col_sums(n, d, one, [&](int i, int j) { return X[int64_t(i) * ld + j] - mean[j]; }, tmp,
                part);
    for (int j = tid; j < d; j += LR_THREADS) scale[j] = tmp[j];    // the correction sum
    __syncthreads();
    lr_col_sums(n, d, one, [&](int i, int j) {
        const double c = X[int64_t(i) * ld + j] - mean[j];
        return c * c;
    }, tmp, part);
    bool bad = false;
    for (int j = tid; j < d; j += LR_THREADS) {
        const double var = (tmp[j] - scale[j] * scale[j] / dn) / dn;
        const double bound = dn * DBL_EPSILON * var + (dn * mean[j] * DBL_EPSILON) *
                                                          (dn * mean[j] * DBL_EPSILON);
        bad |= !isfinite(mean[j]) || !isfinite(var);
        scale[j] = var <= bound ? 1.0 : sqrt(var);
    }
    if (__syncthreads_or(bad) && status == LR_NOT_CONVERGED) status = LR_NONFINITE;
    if (tid == 0) {
        mean[d] = 0.0;
        scale[d] = 1.0;
    }
    for (int j = tid; j < D; j += LR_THREADS) w[j] = 0.0;
    for (int i = tid; i < n; i += LR_THREADS) wx[i] = 0.0;
    __syncthreads();

    // ---- proximal Newton ----------------------------------------------------------------------
    const double tol = LR_TOL * C * dn;
    double F = 0.0, viol = 0.0;
    int it = 0;
    const int col_tiles = (D + LR_TILE - 1) / LR_TILE;
    const int tx = tid % LR_TILE, ty = tid / LR_TILE;
    while (status == LR_NOT_CONVERGED) {
        // loss, gradient weights cg and curvature weights ch at the current margins
        double loss = 0.0;
        for (int i = tid; i < n; i += LR_THREADS) {
            const double s = y[i] * wx[i];
            const double e = exp(-fabs(s));
            loss += lr_loss(s);
            cg[i] = -C * y[i] / (1.0 + exp(s));
            ch[i] = C * e / ((1.0 + e) * (1.0 + e));
        }
        loss = C * lr_block_sum(loss, red);               // (the block sum also fences cg, ch)
        lr_col_sums(n, D, [&](int i) { return cg[i]; }, xt, g, part);
        double pen = 0.0, v = 0.0;
        for (int j = 0; j < D; ++j) pen += l1 ? fabs(w[j]) : 0.5 * w[j] * w[j];
        if (!l1)
            for (int j = tid; j < D; j += LR_THREADS) g[j] += w[j];
        __syncthreads();
        for (int j = tid; j < D; j += LR_THREADS) v = fmax(v, lr_subgrad(g[j], w[j], l1));
        viol = lr_block_max(v, red);
        F = loss + pen;
        if (viol <= tol) {
            status = LR_CONVERGED;
            break;
        }
        if (it == max_iter) break;

        // H = X~^T diag(ch) X~ (+ I for L2, + nu I for L1), lower tiles
        for (int tile = 0; tile < col_tiles * (col_tiles + 1) / 2; ++tile) {
            int ti = 0;
            while ((ti + 1) * (ti + 2) / 2 <= tile) ++ti;
            const int tj = tile - ti * (ti + 1) / 2;
            const int r0 = ti * LR_TILE, c0 = tj * LR_TILE;
            double p[4] = {0.0, 0.0, 0.0, 0.0};
            for (int rb = 0; rb < n; rb += LR_TILE) {
                for (int e = tid; e < LR_TILE * LR_TILE; e += LR_THREADS) {
                    const int ii = e / LR_TILE, cc = e % LR_TILE, i = rb + ii;
                    const int ja = r0 + cc, jb = c0 + cc;
                    A[ii * (LR_TILE + 1) + cc] = (i < n && ja < D) ? xt(i, ja) * ch[i] : 0.0;
                    Bt[ii * (LR_TILE + 1) + cc] = (i < n && jb < D) ? xt(i, jb) : 0.0;
                }
                __syncthreads();
#pragma unroll 8
                for (int ii = 0; ii < LR_TILE; ++ii) {
                    const double b = Bt[ii * (LR_TILE + 1) + tx];
#pragma unroll
                    for (int k = 0; k < 4; ++k)
                        p[k] = fma(A[ii * (LR_TILE + 1) + ty + 8 * k], b, p[k]);
                }
                __syncthreads();
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int row = r0 + ty + 8 * k, col = c0 + tx;
                if (row < D && col <= row)
                    H[row * (row + 1) / 2 + col] = p[k] + (row == col ? (l1 ? LR_NU : 1.0) : 0.0);
            }
        }
        __syncthreads();

        // coordinate descent on g^T delta + delta^T H delta / 2 (+ |w + delta|_1), warp 0
        if (warp == 0) {
            const double inner_tol = fmax(0.01 * viol, 0.1 * tol);
            for (int j = lane; j < D; j += 32) {
                dl[j] = 0.0;
                r[j] = g[j];
            }
            __syncwarp();
            for (int sweep = 0; sweep < LR_MAX_SWEEPS; ++sweep) {
                for (int j = 0; j < D; ++j) {
                    const double hjj = H[j * (j + 1) / 2 + j];
                    const double z = w[j] + dl[j];
                    double zn = z - r[j] / hjj;
                    if (l1) zn = copysign(fmax(fabs(zn) - 1.0 / hjj, 0.0), zn);
                    const double step = zn - z;
                    __syncwarp();
                    if (step != 0.0) {                     // the same value in every lane
                        for (int k = lane; k < D; k += 32) r[k] = fma(H[lr_packed(k, j)], step, r[k]);
                        if (lane == 0) dl[j] = zn - w[j];
                    }
                    __syncwarp();
                }
                double vm = 0.0;
                for (int k = lane; k < D; k += 32) vm = fmax(vm, lr_subgrad(r[k], w[k] + dl[k], l1));
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) vm = fmax(vm, __shfl_xor_sync(0xffffffffu, vm, o));
                if (vm <= inner_tol) break;
            }
            if (lane == 0) {
                // predicted decrease g^T delta + R(w + delta) - R(w) (R = |w|_1 for L1, else 0)
                double pred = 0.0;
                for (int j = 0; j < D; ++j) {
                    pred = fma(g[j], dl[j], pred);
                    if (l1) pred += fabs(w[j] + dl[j]) - fabs(w[j]);
                }
                s_inner = pred;
            }
        }
        __syncthreads();
        const double pred = s_inner;

        // margins of the direction, a warp per row
        for (int i = warp; i < n; i += LR_WARPS) {
            const double* row = X + int64_t(i) * ld;
            double s = 0.0;
            for (int j = lane; j < d; j += 32) s = fma(dl[j], (row[j] - mean[j]) / scale[j], s);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (lane == 0) q[i] = s + dl[d];
        }
        __syncthreads();

        // Armijo line search on F(w + a delta) - F(w); below the rounding level of F the Newton
        // step is taken whole
        double alpha = 1.0;
        bool accepted = pred < 0.0 && -pred <= 1e2 * DBL_EPSILON * F;
        for (int t = 0; !accepted && pred < 0.0 && t < LR_MAX_HALVINGS; ++t) {
            double s = 0.0;
            for (int i = tid; i < n; i += LR_THREADS) {
                const double yi = y[i];
                s += lr_loss(yi * fma(alpha, q[i], wx[i])) - lr_loss(yi * wx[i]);
            }
            double dF = C * lr_block_sum(s, red);
            for (int j = 0; j < D; ++j) {
                const double wn = fma(alpha, dl[j], w[j]);
                dF += l1 ? fabs(wn) - fabs(w[j]) : 0.5 * (wn * wn - w[j] * w[j]);
            }
            if (dF <= LR_ARMIJO * alpha * pred) accepted = true;
            else alpha *= 0.5;
        }
        if (!accepted) break;                              // no decrease: not converged
        for (int i = tid; i < n; i += LR_THREADS) wx[i] = fma(alpha, q[i], wx[i]);
        __syncthreads();
        for (int j = tid; j < D; j += LR_THREADS) w[j] = fma(alpha, dl[j], w[j]);
        __syncthreads();
        ++it;
    }

    if (tid != 0) return;
    const bool failed = status < 0;
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    out[0] = failed ? nan : w[d];
    out[1] = it;
    out[2] = status;
    out[3] = failed ? nan : F;
    out[4] = failed ? nan : viol;
    out[5] = out[6] = out[7] = 0.0;
    for (int j = 0; j < d; ++j) {
        out[LR_HEAD + j] = failed ? nan : mean[j];
        out[LR_HEAD + d + j] = failed ? nan : scale[j];
        out[LR_HEAD + 2 * d + j] = failed ? nan : w[j];
    }
}

__global__ void __launch_bounds__(256)
logreg_predict_kernel(const double* __restrict__ fit, int d, const double* __restrict__ Xq,
                      int64_t ld, int64_t m, double class_min, double* __restrict__ out) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const double* mean = fit + LR_HEAD;
    const double* scale = mean + d;
    const double* coef = scale + d;
    const double* row = Xq + i * ld;
    bool ok = fit[2] >= 0.0;
    double s = 0.0;
    for (int j = 0; j < d; ++j) {
        const double x = row[j];
        ok &= isfinite(x);
        s = fma(coef[j], (x - mean[j]) / scale[j], s);
    }
    const double v = s + fit[0];
    double p = 1.0 / (1.0 + exp(-v));                        // scipy.special.expit
    if (p < class_min) p = class_min;                        // np.maximum (NaN stays NaN)
    out[i] = ok ? log(p / (1.0 - p)) : __longlong_as_double(0x7ff8000000000000ll);
}

}  // namespace elfi

extern "C" {

int elfi_b200_logreg_fit_f64(elfi_b200_ctx* ctx, const double* X, int64_t ld_row, int64_t n,
                             int64_t d, const double* y, int32_t penalty, double C,
                             int64_t max_iter, double* fit, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && X && y && fit, "logreg_fit: NULL argument");
    ELFI_REQUIRE(d >= 1 && d <= LR_D_MAX && n >= 2 && n < (int64_t(1) << 31) && ld_row >= d,
                 "logreg_fit: bad shape (1 <= d <= %d, 2 <= n < 2^31, ld_row >= d; n=%lld d=%lld "
                 "ld_row=%lld)", LR_D_MAX, (long long)n, (long long)d, (long long)ld_row);
    ELFI_REQUIRE(penalty == 0 || penalty == 1,
                 "logreg_fit: penalty must be 0 (L1) or 1 (L2), got %d", int(penalty));
    ELFI_REQUIRE(C > 0.0 && std::isfinite(C), "logreg_fit: C must be positive and finite, got %g",
                 C);
    ELFI_REQUIRE(max_iter >= 0 && max_iter < (int64_t(1) << 31),
                 "logreg_fit: 0 <= max_iter < 2^31, got %lld", (long long)max_iter);
    double* base = static_cast<double*>(ctx_scratch(ctx, size_t(n) * 4 * 8));
    if (!base) return ELFI_B200_ERR_NOMEM;
    const size_t smem = size_t(logreg_smem_doubles(int(d))) * 8;
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        ELFI_CUDA_OK(cudaFuncSetAttribute(logreg_fit_kernel,
                                          cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          int(logreg_smem_doubles(LR_D_MAX) * 8)));
        logreg_fit_kernel<<<1, LR_THREADS, smem, stream>>>(X, ld_row, y, int(n), int(d),
                                                          int(penalty), C, int(max_iter), base,
                                                          base + n, base + 2 * n, base + 3 * n,
                                                          fit);
        return ELFI_B200_OK;
    });
}

int elfi_b200_logreg_predict_f64(elfi_b200_ctx* ctx, const double* fit, int64_t d,
                                 const double* Xq, int64_t ld_row, int64_t m, double class_min,
                                 double* out, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (m == 0 || (fit && Xq && out)), "logreg_predict: NULL argument");
    ELFI_REQUIRE(d >= 1 && d <= LR_D_MAX && m >= 0 && ld_row >= d,
                 "logreg_predict: bad shape (1 <= d <= %d, m >= 0, ld_row >= d; m=%lld d=%lld "
                 "ld_row=%lld)", LR_D_MAX, (long long)m, (long long)d, (long long)ld_row);
    if (m == 0) return ELFI_B200_OK;
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        logreg_predict_kernel<<<unsigned((m + 255) / 256), 256, 0, stream>>>(
            fit, int(d), Xq, ld_row, m, class_min, out);
        return ELFI_B200_OK;
    });
}

}  // extern "C"
