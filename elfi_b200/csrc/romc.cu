// romc.cu -- robust optimisation Monte Carlo (ROMC, elfi/methods/inference/romc.py) in lock-step:
// the Nelder-Mead state machine of every optimisation problem, the line search that bounds each
// solution's acceptance region, uniform draws from the regions with their weights, and the
// unnormalised posterior on a grid of query points.
//
// Problem i is row i of every batch the host evaluates, so one simulator launch serves one point
// of every problem.  Semantics and limits are stated in include/elfi_b200.h.  Arithmetic that has
// to match NumPy uses explicit round-to-nearest intrinsics, so nvcc cannot contract it to FMA.
#include <cmath>

#include "common.cuh"
#include "philox.cuh"

namespace elfi {

constexpr int ROMC_MAX_P = ELFI_B200_ROMC_MAX_P;
constexpr int ROMC_THREADS = 128;
constexpr uint32_t ROMC_SALT = 0x524f4d43u;   // "ROMC": the fourth counter word of the box draws

enum { NM_INIT = 0, NM_REFLECT, NM_EXPAND, NM_CONTRACT_OUT, NM_CONTRACT_IN, NM_SHRINK, NM_DONE };
static_assert(NM_DONE == ELFI_B200_ROMC_NM_DONE, "the header states a finished problem's code");

__host__ __device__ constexpr int64_t nm_state_size(int64_t N) { return (N + 1) * (N + 1) + 3 * N + 2; }

inline unsigned romc_grid(int64_t n) { return unsigned((n + ROMC_THREADS - 1) / ROMC_THREADS); }

// np.argsort's order on a NaN-free prefix, NaN last; ties keep their current order (stable)
__device__ __forceinline__ bool np_less(double a, double b) {
    return a < b || (isnan(b) && !isnan(a));
}

// stable insertion sort of the N + 1 vertices by fsim, rows of sim moved with their values
__device__ __forceinline__ void nm_sort(double* sim, double* fsim, int N) {
    for (int i = 1; i <= N; ++i) {
        for (int j = i; j > 0 && np_less(fsim[j], fsim[j - 1]); --j) {
            const double t = fsim[j];
            fsim[j] = fsim[j - 1];
            fsim[j - 1] = t;
            double* a = sim + j * N;
            double* b = a - N;
#pragma unroll 1
            for (int c = 0; c < N; ++c) {
                const double u = a[c];
                a[c] = b[c];
                b[c] = u;
            }
        }
    }
}

// (The row loops stay rolled: unrolled, ptxas spills the step kernel's state pointers.)
// a * xbar - b * x, one rounding per product and one for the difference
__device__ __forceinline__ void nm_combine(double* dst, const double* xbar, const double* x, double a,
                                           double b, int N) {
#pragma unroll 1
    for (int c = 0; c < N; ++c) dst[c] = __dsub_rn(__dmul_rn(a, xbar[c]), __dmul_rn(b, x[c]));
}

__device__ __forceinline__ void copy_row(double* dst, const double* src, int N) {
#pragma unroll 1
    for (int c = 0; c < N; ++c) dst[c] = src[c];
}

// scipy's initial simplex: x0, then x0 with coordinate k scaled by 1.05 (0.00025 when it is 0)
__global__ void __launch_bounds__(ROMC_THREADS)
romc_nm_init_kernel(int64_t P, int N, const double* __restrict__ x0, int64_t ldx,
                    double* __restrict__ state, int32_t* __restrict__ istate,
                    double* __restrict__ theta, int64_t ldt) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= P) return;
    double* sim = state + i * nm_state_size(N);
    double* fsim = sim + (N + 1) * N;
    const double* x = x0 + i * ldx;
    const double grow = __dadd_rn(1.0, 0.05);
    for (int k = 0; k <= N; ++k) {
        for (int c = 0; c < N; ++c) {
            double v = x[c];
            if (k > 0 && c == k - 1) v = v != 0.0 ? __dmul_rn(grow, v) : 0.00025;
            sim[k * N + c] = v;
        }
        fsim[k] = INFINITY;
    }
    int32_t* st = istate + i * ELFI_B200_ROMC_NM_INTS;
    st[0] = NM_INIT;
    st[1] = 0;   // iterations
    st[2] = 1;   // function evaluations: sim[0] is proposed below
    st[3] = 0;   // vertex being evaluated (initial simplex, shrink)
    st[4] = -1;  // warnflag, set when the problem finishes
    copy_row(theta + i * ldt, sim, N);
}

// One call consumes f at the point each running problem proposed last and advances its state to
// the next point it needs, exactly as scipy's _minimize_neldermead (adaptive=False, no bounds).
__global__ void __launch_bounds__(ROMC_THREADS)
romc_nm_step_kernel(int64_t P, int N, double* __restrict__ state, int32_t* __restrict__ istate,
                    const double* __restrict__ fvals, double* __restrict__ theta, int64_t ldt,
                    int64_t maxiter, int64_t maxfev, double xatol, double fatol) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= P) return;
    int32_t* st = istate + i * ELFI_B200_ROMC_NM_INTS;
    int phase = st[0];
    if (phase == NM_DONE) return;
    int64_t nit = st[1], nfev = st[2];
    int j = st[3];
    double* sim = state + i * nm_state_size(N);
    double* fsim = sim + (N + 1) * N;
    double* xbar = fsim + N + 1;
    double* xr = xbar + N;
    double* xt = xr + N;
    double* fxr = xt + N;          // fxr[0]: f at the reflection; fxr[1]: f_min once done
    double* simN = sim + N * N;
    double* out = theta + i * ldt;
    const double f = fvals[i];
    const double* propose = nullptr;   // the next point, if the problem still runs
    bool end_iteration = false, counted = false, top = false;

    switch (phase) {
        case NM_INIT:
            fsim[j] = f;
            ++j;
            if (j <= N && nfev < maxfev) {
                propose = sim + j * N;
            } else {
                nit = 0;                            // the sort below, then iterations = 1
                end_iteration = counted = true;
            }
            break;
        case NM_REFLECT:
            fxr[0] = f;
            if (f < fsim[0]) {
                nm_combine(xt, xbar, simN, 3.0, 2.0, N);
                phase = NM_EXPAND;
            } else if (f < fsim[N - 1]) {
                copy_row(simN, xr, N);
                fsim[N] = f;
                end_iteration = counted = true;
            } else if (f < fsim[N]) {
                nm_combine(xt, xbar, simN, 1.5, 0.5, N);
                phase = NM_CONTRACT_OUT;
            } else {
                for (int c = 0; c < N; ++c)
                    xt[c] = __dadd_rn(__dmul_rn(0.5, xbar[c]), __dmul_rn(0.5, simN[c]));
                phase = NM_CONTRACT_IN;
            }
            if (!end_iteration) {
                if (nfev < maxfev) propose = xt;
                else end_iteration = true;      // scipy's _MaxFuncCallError: the iteration is not counted
            }
            break;
        case NM_EXPAND:
            if (f < fxr[0]) {
                copy_row(simN, xt, N);
                fsim[N] = f;
            } else {
                copy_row(simN, xr, N);
                fsim[N] = fxr[0];
            }
            end_iteration = counted = true;
            break;
        case NM_CONTRACT_OUT:
        case NM_CONTRACT_IN:
            if (phase == NM_CONTRACT_OUT ? f <= fxr[0] : f < fsim[N]) {
                copy_row(simN, xt, N);
                fsim[N] = f;
                end_iteration = counted = true;
                break;
            }
            j = 0;
            // fall through: shrink towards sim[0], starting with vertex 1
        case NM_SHRINK:
            if (phase == NM_SHRINK) fsim[j] = f;
            phase = NM_SHRINK;
            ++j;
            if (j > N) {
                end_iteration = counted = true;
                break;
            }
            for (int c = 0; c < N; ++c) {
                const double s0 = sim[c];
                sim[j * N + c] = __dadd_rn(s0, __dmul_rn(0.5, __dsub_rn(sim[j * N + c], s0)));
            }
            if (nfev < maxfev) propose = sim + j * N;
            else end_iteration = true;
            break;
    }
    if (end_iteration) {
        if (counted) ++nit;
        nm_sort(sim, fsim, N);
        top = true;
    }
    if (top) {
        bool finish = !(nfev < maxfev && nit < maxiter);
        if (!finish) {
            bool conv = true;
            for (int k = 1; k <= N && conv; ++k)
                for (int c = 0; c < N; ++c)
                    if (!(fabs(__dsub_rn(sim[k * N + c], sim[c])) <= xatol)) conv = false;
            for (int k = 1; k <= N && conv; ++k)
                if (!(fabs(__dsub_rn(fsim[0], fsim[k])) <= fatol)) conv = false;
            finish = conv;
        }
        if (finish) {
            double fmin = fsim[0];
            for (int k = 0; k <= N; ++k) {
                if (isnan(fsim[k])) fmin = fsim[k];
                else if (!isnan(fmin) && fsim[k] < fmin) fmin = fsim[k];
            }
            fxr[1] = fmin;
            st[4] = nfev >= maxfev ? 1 : (nit >= maxiter ? 2 : 0);
            phase = NM_DONE;
            copy_row(out, sim, N);
        } else {
            for (int c = 0; c < N; ++c) {
                double s = sim[c];
                for (int k = 1; k < N; ++k) s = __dadd_rn(s, sim[k * N + c]);
                xbar[c] = __ddiv_rn(s, double(N));
            }
            nm_combine(xr, xbar, simN, 2.0, 1.0, N);
            phase = NM_REFLECT;
            propose = xr;
        }
    }
    if (propose) {
        copy_row(out, propose, N);
        ++nfev;
    }
    st[0] = phase;
    st[1] = int32_t(nit);
    st[2] = int32_t(nfev);
    st[3] = j;
}

// ---- line search along the rotated axes (romc.py line_search) ----------------------------------
// pair dp = 2 d + side: direction d (column d of the rotation), side 0 along -v_d, side 1 along v_d.
// Per pair: th (N), offset, eta; ints: refinement, repetitions, done.
__global__ void __launch_bounds__(ROMC_THREADS)
romc_line_search_kernel(int init, int64_t P, int N, const double* __restrict__ x_min,
                        const double* __restrict__ rot, const int32_t* __restrict__ active,
                        double* __restrict__ state, int32_t* __restrict__ istate,
                        const double* __restrict__ fvals, double* __restrict__ theta, double eps,
                        int K, double eta0, int rep_lim, double* __restrict__ limits) {
    const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (t >= 2 * N * P) return;
    const int dp = int(t / P);
    const int64_t i = t - dp * P;
    const int d = dp >> 1, side = dp & 1;
    double* th = state + t * (N + 2);
    double& offset = th[N];
    double& eta = th[N + 1];
    int32_t* st = istate + t * 4;
    double* out = theta + t * N;
    if (init) {
        copy_row(th, x_min + i * N, N);
        offset = 0.0;
        eta = eta0;
        st[0] = 0;
        st[1] = 0;
        st[2] = active[i] ? 0 : 1;
        copy_row(out, th, N);
        return;
    }
    if (st[2]) return;
    const double* R = rot + i * N * N;
    const double f = fvals[t];
    int k = st[0], rep = st[1];
    bool done = false;
    if (f < eps && rep <= rep_lim) {
        for (int c = 0; c < N; ++c) {
            const double v = side ? R[c * N + d] : -R[c * N + d];
            th[c] = __dadd_rn(th[c], __dmul_rn(eta, v));
        }
        offset = __dadd_rn(offset, eta);
        ++rep;
    } else {
        for (int c = 0; c < N; ++c) {
            const double v = side ? R[c * N + d] : -R[c * N + d];
            th[c] = __dsub_rn(th[c], __dmul_rn(eta, v));
        }
        offset = __dsub_rn(offset, eta);
        if (rep > rep_lim) {
            done = true;
        } else {
            eta = __ddiv_rn(eta, 2.0);
            ++k;
            rep = 0;
            done = k >= K;
        }
    }
    if (done) {
        if (offset <= 0.0) offset = eta;
        limits[(i * N + d) * 2 + side] = side ? offset : -offset;
        st[2] = 1;
    }
    st[0] = k;
    st[1] = rep;
    copy_row(out, th, N);
}

// ---- regions: containment and the local quadratic surrogate ------------------------------------
// rotation_inv @ x + rotation_inv @ (-center), each product summed over the columns in order
__device__ __forceinline__ bool box_contains(const double (&x)[ROMC_MAX_P], const double* Rinv,
                                             const double* c, const double* lim, int N) {
    bool inside = true;
    for (int r = 0; r < N; ++r) {
        double a = 0.0, b = 0.0;
#pragma unroll
        for (int k = 0; k < ROMC_MAX_P; ++k) {
            if (k < N) {
                a = __dadd_rn(a, __dmul_rn(Rinv[r * N + k], x[k]));
                b = __dadd_rn(b, __dmul_rn(Rinv[r * N + k], -c[k]));
            }
        }
        const double y = __dadd_rn(a, b);
        if (y < lim[2 * r] || y > lim[2 * r + 1]) inside = false;
    }
    return inside;
}

// PolynomialFeatures(degree=2) @ coef: 1, x_i, then x_i x_j for i <= j, summed in that order
__device__ __forceinline__ double quad_surrogate(const double (&x)[ROMC_MAX_P], const double* coef,
                                                int N) {
    double s = coef[0];
#pragma unroll
    for (int a = 0; a < ROMC_MAX_P; ++a)
        if (a < N) s = __dadd_rn(s, __dmul_rn(coef[1 + a], x[a]));
    int e = 1 + N;
#pragma unroll
    for (int a = 0; a < ROMC_MAX_P; ++a) {
#pragma unroll
        for (int b = a; b < ROMC_MAX_P; ++b) {
            if (b < N) s = __dadd_rn(s, __dmul_rn(coef[e++], __dmul_rn(x[a], x[b])));
        }
    }
    return s;
}

__global__ void __launch_bounds__(ROMC_THREADS)
romc_box_sample_kernel(int64_t R, int N, int64_t n2, const double* __restrict__ center,
                       const double* __restrict__ rot, const double* __restrict__ rot_inv,
                       const double* __restrict__ lim, const double* __restrict__ volume,
                       uint64_t seed, const double* __restrict__ coef, int64_t ncoef,
                       double* __restrict__ pts, double* __restrict__ q, double* __restrict__ surr) {
    const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (t >= R * n2) return;
    const int64_t r = t / n2, jj = t - r * n2;
    const double* L = lim + r * N * 2;
    const double* Rm = rot + r * N * N;
    const double* c = center + r * N;
    const Philox gen(seed);
    double u[ROMC_MAX_P], x[ROMC_MAX_P];
#pragma unroll
    for (int d = 0; d < ROMC_MAX_P; d += 2) {
        if (d < N) {
            const PhiloxWords w = gen(uint32_t(jj), uint32_t(r), uint32_t(d >> 1), ROMC_SALT);
            u[d] = __dadd_rn(L[2 * d], __dmul_rn(__dsub_rn(L[2 * d + 1], L[2 * d]), u01(w.x, w.y)));
            if (d + 1 < N)
                u[d + 1] = __dadd_rn(L[2 * d + 2],
                                     __dmul_rn(__dsub_rn(L[2 * d + 3], L[2 * d + 2]), u01(w.z, w.w)));
        }
    }
    double* out = pts + t * N;
#pragma unroll
    for (int a = 0; a < ROMC_MAX_P; ++a) {
        x[a] = 0.0;
        if (a < N) {
            double s = 0.0;
#pragma unroll
            for (int b = 0; b < ROMC_MAX_P; ++b)
                if (b < N) s = __dadd_rn(s, __dmul_rn(Rm[a * N + b], u[b]));
            x[a] = __dadd_rn(s, c[a]);
            out[a] = x[a];
        }
    }
    q[t] = box_contains(x, rot_inv + r * N * N, c, L, N) ? __ddiv_rn(1.0, volume[r]) : 0.0;
    if (surr) surr[t] = quad_surrogate(x, coef + r * ncoef, N);
}

__global__ void __launch_bounds__(ROMC_THREADS)
romc_weights_kernel(int64_t n, const double* __restrict__ dist, const double* __restrict__ prior,
                    const double* __restrict__ q, double eps, double* __restrict__ w) {
    const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const double qt = q[t];
    w[t] = qt > 0.0 ? __ddiv_rn(__dmul_rn(dist[t] < eps ? 1.0 : 0.0, prior[t]), qt) : 0.0;
}

__global__ void __launch_bounds__(ROMC_THREADS)
romc_posterior_unnorm_kernel(int64_t M, int64_t R, int N, const double* __restrict__ theta,
                             int64_t ldt, const double* __restrict__ center,
                             const double* __restrict__ rot_inv, const double* __restrict__ lim,
                             const double* __restrict__ coef, int64_t ncoef,
                             const double* __restrict__ fvals, int64_t ldf, double eps,
                             const double* __restrict__ prior, double* __restrict__ out) {
    const int64_t m = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (m >= M) return;
    double x[ROMC_MAX_P];
#pragma unroll
    for (int a = 0; a < ROMC_MAX_P; ++a) x[a] = a < N ? theta[m * ldt + a] : 0.0;
    int64_t count = 0;
    for (int64_t k = 0; k < R; ++k) {
        if (fvals) {
            count += fvals[m * ldf + k] <= eps;
        } else if (box_contains(x, rot_inv + k * N * N, center + k * N, lim + k * N * 2, N)) {
            count += quad_surrogate(x, coef + k * ncoef, N) <= eps;
        }
    }
    out[m] = __dmul_rn(prior[m], double(count));
}

}  // namespace elfi

extern "C" {

int elfi_b200_romc_nm_init_f64(elfi_b200_ctx* ctx, int64_t P, int64_t p, const double* x0,
                               int64_t ld_x0, double* state, int32_t* istate, double* theta,
                               int64_t ld_theta, void* stream) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (P == 0 || (x0 && state && istate && theta)), "romc_nm_init: NULL argument");
    ELFI_REQUIRE(p >= 1 && p <= ROMC_MAX_P && P >= 0 && P < (int64_t(1) << 31) && ld_x0 >= p &&
                     ld_theta >= p,
                 "romc_nm_init: bad shape (1 <= p <= %d, 0 <= P < 2^31, ld_x0 >= p, ld_theta >= p; "
                 "p=%lld P=%lld ld_x0=%lld ld_theta=%lld)", ROMC_MAX_P, (long long)p, (long long)P,
                 (long long)ld_x0, (long long)ld_theta);
    if (P == 0) return ELFI_B200_OK;
    return run_on_device(ctx, stream, [&](cudaStream_t s) {
        romc_nm_init_kernel<<<romc_grid(P), ROMC_THREADS, 0, s>>>(P, int(p), x0, ld_x0, state, istate,
                                                                  theta, ld_theta);
        return ELFI_B200_OK;
    });
}

int elfi_b200_romc_nm_step_f64(elfi_b200_ctx* ctx, int64_t P, int64_t p, double* state,
                               int32_t* istate, const double* fvals, double* theta,
                               int64_t ld_theta, int64_t maxiter, int64_t maxfev, double xatol,
                               double fatol, void* stream) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (P == 0 || (state && istate && fvals && theta)),
                 "romc_nm_step: NULL argument");
    ELFI_REQUIRE(p >= 1 && p <= ROMC_MAX_P && P >= 0 && P < (int64_t(1) << 31) && ld_theta >= p,
                 "romc_nm_step: bad shape (1 <= p <= %d, 0 <= P < 2^31, ld_theta >= p; p=%lld "
                 "P=%lld ld_theta=%lld)", ROMC_MAX_P, (long long)p, (long long)P,
                 (long long)ld_theta);
    ELFI_REQUIRE(maxiter >= 1 && maxiter < (int64_t(1) << 30) && maxfev >= 1 &&
                     maxfev < (int64_t(1) << 30) && xatol >= 0 && fatol >= 0,
                 "romc_nm_step: need 1 <= maxiter, maxfev < 2^30 and xatol, fatol >= 0");
    if (P == 0) return ELFI_B200_OK;
    return run_on_device(ctx, stream, [&](cudaStream_t s) {
        romc_nm_step_kernel<<<romc_grid(P), ROMC_THREADS, 0, s>>>(P, int(p), state, istate, fvals,
                                                                  theta, ld_theta, maxiter, maxfev,
                                                                  xatol, fatol);
        return ELFI_B200_OK;
    });
}

int elfi_b200_romc_line_search_f64(elfi_b200_ctx* ctx, int32_t init, int64_t P, int64_t p,
                                   const double* x_min, const double* rot, const int32_t* active,
                                   double* state, int32_t* istate, const double* fvals,
                                   double* theta, double eps, int64_t K, double eta,
                                   int64_t rep_lim, double* limits, void* stream) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (P == 0 || (x_min && rot && active && state && istate && theta && limits &&
                                    (init || fvals))),
                 "romc_line_search: NULL argument");
    ELFI_REQUIRE(p >= 1 && p <= ROMC_MAX_P && P >= 0 && 2 * p * P < (int64_t(1) << 31),
                 "romc_line_search: bad shape (1 <= p <= %d, 0 <= 2 p P < 2^31; p=%lld P=%lld)",
                 ROMC_MAX_P, (long long)p, (long long)P);
    ELFI_REQUIRE(K >= 1 && K < (int64_t(1) << 30) && rep_lim >= 0 && rep_lim < (int64_t(1) << 30) &&
                     eta > 0 && std::isfinite(eta),
                 "romc_line_search: need 1 <= K < 2^30, 0 <= rep_lim < 2^30 and a finite eta > 0");
    if (P == 0) return ELFI_B200_OK;
    return run_on_device(ctx, stream, [&](cudaStream_t s) {
        romc_line_search_kernel<<<romc_grid(2 * p * P), ROMC_THREADS, 0, s>>>(
            init, P, int(p), x_min, rot, active, state, istate, fvals, theta, eps, int(K), eta,
            int(rep_lim), limits);
        return ELFI_B200_OK;
    });
}

int elfi_b200_romc_box_sample_f64(elfi_b200_ctx* ctx, int64_t R, int64_t p, int64_t n2,
                                  const double* center, const double* rot, const double* rot_inv,
                                  const double* limits, const double* volume, uint64_t seed,
                                  const double* coef, double* pts, double* q, double* surr,
                                  void* stream) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (R * n2 == 0 || (center && rot && rot_inv && limits && volume && pts && q)) &&
                     (!surr || coef),
                 "romc_box_sample: NULL argument");
    ELFI_REQUIRE(p >= 1 && p <= ROMC_MAX_P && R >= 0 && R < (int64_t(1) << 31) && n2 >= 0 &&
                     n2 < (int64_t(1) << 31) && R * n2 < (int64_t(1) << 40),
                 "romc_box_sample: bad shape (1 <= p <= %d, 0 <= R, n2 < 2^31, R n2 < 2^40; p=%lld "
                 "R=%lld n2=%lld)", ROMC_MAX_P, (long long)p, (long long)R, (long long)n2);
    if (R * n2 == 0) return ELFI_B200_OK;
    const int64_t nc = 1 + p + p * (p + 1) / 2;
    return run_on_device(ctx, stream, [&](cudaStream_t s) {
        romc_box_sample_kernel<<<romc_grid(R * n2), ROMC_THREADS, 0, s>>>(
            R, int(p), n2, center, rot, rot_inv, limits, volume, seed, coef, nc, pts, q, surr);
        return ELFI_B200_OK;
    });
}

int elfi_b200_romc_weights_f64(elfi_b200_ctx* ctx, int64_t n, const double* dist,
                               const double* prior, const double* q, double eps, double* w,
                               void* stream) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (n == 0 || (dist && prior && q && w)), "romc_weights: NULL argument");
    ELFI_REQUIRE(n >= 0 && n < (int64_t(1) << 40), "romc_weights: bad length %lld", (long long)n);
    if (n == 0) return ELFI_B200_OK;
    return run_on_device(ctx, stream, [&](cudaStream_t s) {
        romc_weights_kernel<<<romc_grid(n), ROMC_THREADS, 0, s>>>(n, dist, prior, q, eps, w);
        return ELFI_B200_OK;
    });
}

int elfi_b200_romc_posterior_unnorm_f64(elfi_b200_ctx* ctx, int64_t M, int64_t R, int64_t p,
                                        const double* theta, int64_t ld_theta,
                                        const double* center, const double* rot_inv,
                                        const double* limits, const double* coef,
                                        const double* fvals, int64_t ld_f, double eps,
                                        const double* prior, double* out, void* stream) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (M == 0 || (theta && prior && out)) &&
                     (R == 0 || fvals || (center && rot_inv && limits && coef)),
                 "romc_posterior_unnorm: NULL argument");
    ELFI_REQUIRE(p >= 1 && p <= ROMC_MAX_P && M >= 0 && M < (int64_t(1) << 40) && R >= 0 &&
                     R < (int64_t(1) << 31) && ld_theta >= p && (!fvals || ld_f >= R),
                 "romc_posterior_unnorm: bad shape (1 <= p <= %d, 0 <= M < 2^40, 0 <= R < 2^31, "
                 "ld_theta >= p, ld_f >= R; p=%lld M=%lld R=%lld)", ROMC_MAX_P, (long long)p,
                 (long long)M, (long long)R);
    if (M == 0) return ELFI_B200_OK;
    const int64_t nc = 1 + p + p * (p + 1) / 2;
    return run_on_device(ctx, stream, [&](cudaStream_t s) {
        romc_posterior_unnorm_kernel<<<romc_grid(M), ROMC_THREADS, 0, s>>>(
            M, R, int(p), theta, ld_theta, center, rot_inv, limits, coef, nc, fvals, ld_f, eps,
            prior, out);
        return ELFI_B200_OK;
    });
}

}  // extern "C"
