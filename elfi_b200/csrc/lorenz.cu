// lorenz.cu -- the Lorenz forecast model of elfi/examples/lorenz.py in throughput mode: the
// stochastic Lorenz 96 simulator (a 40-variable ring integrated by RK4 with AR(1) forcing) and its
// six summaries [Mean, Var, Autocov, Cov, CrosscovPrev, CrosscovNext], alone or fused.
//
// Random stream (Philox4x32-10 keyed by the seed; counter (row, row >> 32, block, salt)):
//   sim_lorenz  row = offset + i; the normal e of step s (1 <= s < n_timestep) and variable k is
//               Box-Muller normal (k & 1) of block (s << 6) | (k >> 1) (boxmuller.cuh)
// so every draw is a pure function of (seed, offset + row, s, k), whatever the lane layout.
//
// Model (lorenz.py:94-163): row 0 is the initial state, then for s = 1 .. n_timestep - 1
//   eta = phi * eta + e * sqrt(1 - phi^2)   (eta starts at 0; sqrt(1 - phi^2) comes from the host)
//   y = RK4 step of dy_k/dt = -y[k-2] y[k-1] + y[k-1] y[k+1] - y[k] + f - (theta1 + y[k] theta2) + eta[k]
// with the arithmetic of lorenz.cuh (the reference's order, no FMA, a real division by 6).
//
// Layout: a row's m variables are spread over L = ceil(m / V) consecutive lanes, V in {1, 2, 4}
// variables per lane (lane l holds k = l V .. l V + V - 1; the last lane may hold fewer), and a warp
// takes floor(32 / L) rows (for m = 40: V = 4, L = 10, 3 rows, 30 lanes busy).  y, the stage input,
// the RK4 accumulator and eta stay in registers; the neighbours k - 2, k - 1, k + 1 of a lane's
// first and last variables come from the lanes before and after it in the row's segment by
// __shfl_sync (three shuffles per derivative, four when the last lane holds one variable).
//
// Summaries (2 <= m: with one variable NumPy sums the time axis pairwise): one warp per row.  Lanes
// take columns for the sums over time (sequential in t, as
// NumPy adds along a non-contiguous axis), then groups of 8 lanes take NumPy's pairwise sums over
// the flattened row leaf by leaf: lane c of a group runs accumulator c of a leaf, three xor
// shuffles give the fold, and PairwiseLeaves (lorenz.cuh) combines the leaves in NumPy's order.
// The fused kernel simulates a warp's rows into a slab of global scratch (R * T * m doubles per
// resident warp, independent of B) and summarises the slab with the same code: the bits of
// sim_lorenz followed by lorenz_summaries.
#include "boxmuller.cuh"
#include "common.cuh"
#include "lorenz.cuh"
#include "philox.cuh"

namespace elfi {

constexpr uint32_t SALT_LORENZ = 0x4c4f525au;   // "LORZ"
constexpr int LORENZ_M_MIN = ELFI_B200_LORENZ_NOBS_MIN;
constexpr int LORENZ_M_MAX = ELFI_B200_LORENZ_NOBS_MAX;
constexpr int64_t LORENZ_T_MAX = ELFI_B200_LORENZ_T_MAX;   // s << 6 fits the 32-bit block word
constexpr int LORENZ_THREADS = 128;
constexpr int LORENZ_WARPS = LORENZ_THREADS / 32;
constexpr int LORENZ_FUSED_BLOCKS_PER_SM = 4;
constexpr size_t LORENZ_SLAB_BUDGET = size_t(512) << 20;   // bytes of fused scratch at most

struct LorenzSim {
    const double* P;
    int64_t ldP;
    int64_t B;
    int m, T;
    const double* init;
    double f, phi, s, dt;
    uint64_t seed, offset;
};

// y[i] for a run-time i without an indexed (local-memory) access
template <int V>
__device__ __forceinline__ double pick(const double (&y)[V], int i) {
    double r = y[0];
#pragma unroll
    for (int v = 1; v < V; ++v)
        if (i == v) r = y[v];
    return r;
}

// k[v] = dt * dy/dt at the stage st (the lane's V variables of one row)
template <int V>
__device__ __forceinline__ void lorenz_ode(const LorenzSim& a, const double (&st)[V],
                                           const double (&eta)[V], double th1, double th2, int nv,
                                           int prev, int prev2, int next, bool prev_has_one,
                                           double (&k)[V]) {
    double h1, h2, hr;
    if (V == 1) {
        h1 = __shfl_sync(0xffffffffu, st[0], prev);
        h2 = __shfl_sync(0xffffffffu, st[0], prev2);
        hr = __shfl_sync(0xffffffffu, st[0], next);
    } else {
        const double p1 = pick(st, nv - 1), p2 = pick(st, nv - 2 < 0 ? 0 : nv - 2);
        h1 = __shfl_sync(0xffffffffu, p1, prev);
        h2 = __shfl_sync(0xffffffffu, p2, prev);
        hr = __shfl_sync(0xffffffffu, st[0], next);
        if (a.m % V == 1) {   // the last lane holds one variable: k - 2 of lane 0 is two lanes back
            const double h2b = __shfl_sync(0xffffffffu, p1, prev2);
            if (prev_has_one) h2 = h2b;
        }
    }
#pragma unroll
    for (int v = 0; v < V; ++v) {
        const double ym1 = v >= 1 ? st[v >= 1 ? v - 1 : 0] : h1;
        const double ym2 = v >= 2 ? st[v >= 2 ? v - 2 : 0] : (v == 1 ? h1 : h2);
        const double yp1 = (v + 1 < nv) ? st[v + 1 < V ? v + 1 : 0] : hr;
        k[v] = __dmul_rn(a.dt, lorenz_deriv(ym2, ym1, st[v], yp1, a.f, th1, th2, eta[v]));
    }
}

// Simulates the row of this lane's segment into dst[t * m + k] (row-major (T, m) at dst; NULL for
// lanes without a row).  Every lane of the warp calls it (the shuffles need the whole warp).
template <int V>
__device__ __forceinline__ void lorenz_sim_row(const LorenzSim& a, int L, int64_t row, bool live,
                                               double* dst, int64_t ldt) {
    const int lane = threadIdx.x & 31;
    const int seg = lane / L, ll = lane - seg * L;
    const int base = seg * L;
    const int prev = base + (ll + L - 1) % L, prev2 = base + (ll + L - 2) % L,
              next = base + (ll + 1) % L;
    const int k0 = ll * V;
    int nv = a.m - k0;
    if (nv > V) nv = V;
    const bool prev_has_one = (ll == 0) && (a.m % V == 1);
    const double th1 = live ? a.P[row * a.ldP] : 0.0;
    const double th2 = live ? a.P[row * a.ldP + 1] : 0.0;
    const Philox ph(a.seed);
    const uint64_t crow = a.offset + uint64_t(row);
    const uint32_t r0 = uint32_t(crow), r1 = uint32_t(crow >> 32);
    double y[V], eta[V], st[V], acc[V], k[V];
#pragma unroll
    for (int v = 0; v < V; ++v) {
        y[v] = (v < nv) ? a.init[k0 + v] : 0.0;
        eta[v] = 0.0;
        if (live && v < nv) dst[k0 + v] = y[v];
    }
    for (int s = 1; s < a.T; ++s) {
        const uint32_t blk = uint32_t(s) << 6;
        if (V == 1) {
            double n0, n1;
            normal2(ph(r0, r1, blk | uint32_t(k0 >> 1), SALT_LORENZ), n0, n1);
            eta[0] = lorenz_ar1(eta[0], (k0 & 1) ? n1 : n0, a.phi, a.s);
        } else {
#pragma unroll
            for (int v = 0; v < V; v += 2) {
                if (v < nv) {
                    double n0, n1;
                    normal2(ph(r0, r1, blk | uint32_t((k0 + v) >> 1), SALT_LORENZ), n0, n1);
                    eta[v] = lorenz_ar1(eta[v], n0, a.phi, a.s);
                    eta[v + 1] = lorenz_ar1(eta[v + 1], n1, a.phi, a.s);
                }
            }
        }
        lorenz_ode<V>(a, y, eta, th1, th2, nv, prev, prev2, next, prev_has_one, k);
#pragma unroll
        for (int v = 0; v < V; ++v) {
            acc[v] = k[v];
            st[v] = lorenz_half_stage(y[v], k[v]);
        }
        lorenz_ode<V>(a, st, eta, th1, th2, nv, prev, prev2, next, prev_has_one, k);
#pragma unroll
        for (int v = 0; v < V; ++v) {
            acc[v] = __dadd_rn(acc[v], __dmul_rn(2.0, k[v]));
            st[v] = lorenz_half_stage(y[v], k[v]);
        }
        lorenz_ode<V>(a, st, eta, th1, th2, nv, prev, prev2, next, prev_has_one, k);
#pragma unroll
        for (int v = 0; v < V; ++v) {
            acc[v] = __dadd_rn(acc[v], __dmul_rn(2.0, k[v]));
            st[v] = __dadd_rn(y[v], k[v]);
        }
        lorenz_ode<V>(a, st, eta, th1, th2, nv, prev, prev2, next, prev_has_one, k);
#pragma unroll
        for (int v = 0; v < V; ++v) {
            y[v] = __dadd_rn(y[v], __ddiv_rn(__dadd_rn(acc[v], k[v]), 6.0));
            if (live && v < nv) dst[int64_t(s) * ldt + k0 + v] = y[v];
        }
    }
}

// ---------------------------------------------------------------------------- summaries
// Sum of NumPy's pairwise order over n terms, four channels at once: the group g = lane / 8 sums
// term(g, t, k) over j = t * m + k < n (all lanes of a group return the channel's sum).
template <class Term>
__device__ __forceinline__ double warp_pairwise(int n, int m, const Term& term) {
    const int c = threadIdx.x & 7;
    PairwiseLeaves<LORENZ_SUMM_MAXD> w;
    w.begin(n);
    for (;;) {
        const int s = w.start, L = w.len;
        const int L8 = (L < 8) ? 0 : L - L % 8;
        double v = 0.0;
        if (L8 > 0) {
            int j = s + c;
            int t = j / m, k = j - t * m;
            v = term(t, k);
            for (int i = 8 + c; i < L8; i += 8) {
                k += 8;
                while (k >= m) {
                    k -= m;
                    ++t;
                }
                v = __dadd_rn(v, term(t, k));
            }
            v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, 1));
            v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, 2));
            v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, 4));
        }
        if (L8 < L) {
            int j = s + L8;
            int t = j / m, k = j - t * m;
            for (int i = L8; i < L; ++i) {
                v = __dadd_rn(v, term(t, k));
                if (++k == m) {
                    k = 0;
                    ++t;
                }
            }
        }
        if (!w.add_leaf(v)) break;
    }
    return w.total();
}

// The six summaries of the row x[t * ldt + k * ldk] (T, m); every lane of the warp calls it and
// gets them in out[6].  sm: 5 * LORENZ_M_MAX doubles of this warp's shared memory.
__device__ __forceinline__ void warp_row_summaries(const double* __restrict__ x, int64_t ldt,
                                                   int64_t ldk, int T, int m, double* sm,
                                                   double (&out)[6]) {
    const int lane = threadIdx.x & 31;
    const int g = lane >> 3;
    double* M = sm;
    double* A = sm + LORENZ_M_MAX;
    double* Bm = sm + 2 * LORENZ_M_MAX;
    double* Vc = sm + 3 * LORENZ_M_MAX;
    double* Cc = sm + 4 * LORENZ_M_MAX;
    auto X = [&](int t, int k) { return x[int64_t(t) * ldt + int64_t(k) * ldk]; };
    for (int k = lane; k < m; k += 32) {
        double sa = 0.0, sb = 0.0;
        for (int t = 0; t < T - 1; ++t) {
            sa = __dadd_rn(sa, X(t, k));
            sb = __dadd_rn(sb, X(t + 1, k));
        }
        M[k] = __ddiv_rn(__dadd_rn(sa, X(T - 1, k)), double(T));
        A[k] = __ddiv_rn(sa, double(T - 1));
        Bm[k] = __ddiv_rn(sb, double(T - 1));
    }
    __syncwarp();
    for (int k = lane; k < m; k += 32) {
        const int kr = (k + 1 == m) ? 0 : k + 1;
        const double mk = M[k], mr = M[kr];
        double v = 0.0, c = 0.0;
        for (int t = 0; t < T; ++t) {
            const double d = __dsub_rn(X(t, k), mk);
            v = __dadd_rn(v, __dmul_rn(d, d));
            c = __dadd_rn(c, __dmul_rn(d, __dsub_rn(X(t, kr), mr)));
        }
        Vc[k] = __ddiv_rn(v, double(T));
        Cc[k] = __ddiv_rn(c, double(T));
    }
    __syncwarp();
    // np.mean over space of the column variances (group 0) and covariances (group 1)
    const double* col = (g & 1) ? Cc : Vc;
    const double sp = warp_pairwise(m, m, [&](int, int k) { return col[k]; });
    // Autocov (group 0), CrosscovPrev (group 1), CrosscovNext (group 2; group 3 repeats group 0)
    const int dk = (g == 1) ? m - 1 : (g == 2) ? 1 : 0;
    const double cr = warp_pairwise((T - 1) * m, m, [&](int t, int k) {
        int kk = k + dk;
        if (kk >= m) kk -= m;
        return lorenz_cross(X(t, k), A[k], X(t + 1, kk), Bm[kk]);
    });
    const double mean = warp_pairwise(T * m, m, [&](int t, int k) { return X(t, k); });
    const double n1 = double((T - 1) * m);
    out[0] = __ddiv_rn(mean, double(T * m));
    out[1] = __ddiv_rn(__shfl_sync(0xffffffffu, sp, 0), double(m));
    out[2] = __ddiv_rn(__shfl_sync(0xffffffffu, cr, 0), n1);
    out[3] = __ddiv_rn(__shfl_sync(0xffffffffu, sp, 8), double(m));
    out[4] = __ddiv_rn(__shfl_sync(0xffffffffu, cr, 8), n1);
    out[5] = __ddiv_rn(__shfl_sync(0xffffffffu, cr, 16), n1);
    __syncwarp();   // sm is reused by the next row
}

// ---------------------------------------------------------------------------- kernels
// One warp per group of R = 32 / L rows; X (B, T, m) C-contiguous.
template <int V>
__global__ void __launch_bounds__(LORENZ_THREADS)
sim_lorenz_kernel(const LorenzSim a, int L, int R, int64_t n_groups, double* __restrict__ X) {
    const int64_t group = int64_t(blockIdx.x) * LORENZ_WARPS + (threadIdx.x >> 5);
    if (group >= n_groups) return;   // whole warps only
    const int seg = (threadIdx.x & 31) / L;
    const int64_t row = group * R + seg;
    const bool live = seg < R && row < a.B;
    const int64_t tm = int64_t(a.T) * a.m;
    lorenz_sim_row<V>(a, L, row, live, live ? X + row * tm : nullptr, a.m);
}

// One warp per row, grid-stride.
__global__ void __launch_bounds__(LORENZ_THREADS)
lorenz_summaries_kernel(const double* __restrict__ X, int64_t ld_row, int64_t ld_t, int64_t ld_k,
                        int64_t B, int T, int m, double* __restrict__ S, int64_t ldS) {
    __shared__ double sm_all[LORENZ_WARPS][5 * LORENZ_M_MAX];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int64_t row = int64_t(blockIdx.x) * LORENZ_WARPS + warp; row < B;
         row += int64_t(gridDim.x) * LORENZ_WARPS) {
        double out[6];
        warp_row_summaries(X + row * ld_row, ld_t, ld_k, T, m, sm_all[warp], out);
        if (lane < 6) {
            double o = out[0];
#pragma unroll
            for (int j = 1; j < 6; ++j)
                if (lane == j) o = out[j];
            S[row * ldS + lane] = o;
        }
    }
}

// Fused: each warp simulates its R rows into its slab (R * T * m doubles of scratch) and
// summarises them from there; grid-stride over the row groups.  Without the minimum of 4 blocks
// per SM ptxas settles on 96 registers and spills 40 B; with it, 128 registers and no spill.
template <int V>
__global__ void __launch_bounds__(LORENZ_THREADS, LORENZ_FUSED_BLOCKS_PER_SM)
sim_lorenz_fused_kernel(const LorenzSim a, int L, int R, int64_t n_groups, double* __restrict__ slab_all,
                        double* __restrict__ S, int64_t ldS) {
    __shared__ double sm_all[LORENZ_WARPS][5 * LORENZ_M_MAX];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t tm = int64_t(a.T) * a.m;
    const int64_t gw = int64_t(blockIdx.x) * LORENZ_WARPS + warp;
    double* slab = slab_all + gw * R * tm;
    const int seg = lane / L;
    for (int64_t group = gw; group < n_groups; group += int64_t(gridDim.x) * LORENZ_WARPS) {
        const int64_t row0 = group * R;
        const bool live = seg < R && row0 + seg < a.B;
        lorenz_sim_row<V>(a, L, row0 + seg, live, live ? slab + seg * tm : nullptr, a.m);
        __syncwarp();
        for (int r = 0; r < R && row0 + r < a.B; ++r) {
            double out[6];
            warp_row_summaries(slab + r * tm, a.m, 1, a.T, a.m, sm_all[warp], out);
            if (lane < 6) {
                double o = out[0];
#pragma unroll
                for (int j = 1; j < 6; ++j)
                    if (lane == j) o = out[j];
                S[(row0 + r) * ldS + lane] = o;
            }
        }
        __syncwarp();   // the slab is rewritten by the next group
    }
}

// V in {1, 2, 4} with L = ceil(m / V) <= 32 that keeps the most lanes busy (ties: the smaller V)
static int lorenz_vars_per_lane(int m) {
    int best = 0;
    double best_util = -1.0;
    for (int V : {1, 2, 4}) {
        const int L = (m + V - 1) / V;
        if (L > 32) continue;
        const double util = double((32 / L) * m) / double(32 * V);
        if (util > best_util) {
            best_util = util;
            best = V;
        }
    }
    return best;
}

template <int V>
static int launch_sim_lorenz(elfi_b200_ctx* ctx, const LorenzSim& a, double* X, double* S,
                             int64_t ldS, cudaStream_t stream) {
    const int L = (a.m + V - 1) / V, R = 32 / L;
    const int64_t n_groups = (a.B + R - 1) / R;
    if (X) {
        const int64_t blocks = (n_groups + LORENZ_WARPS - 1) / LORENZ_WARPS;
        sim_lorenz_kernel<V><<<unsigned(blocks), LORENZ_THREADS, 0, stream>>>(a, L, R, n_groups, X);
        ELFI_CUDA_OK(cudaGetLastError());
        if (S) {
            const unsigned sb = capped_grid(ctx, a.B, LORENZ_WARPS, 16);
            const int64_t tm = int64_t(a.T) * a.m;
            lorenz_summaries_kernel<<<sb, LORENZ_THREADS, 0, stream>>>(
                X, tm, a.m, 1, a.B, a.T, a.m, S, ldS);
        }
        return ELFI_B200_OK;
    }
    const size_t slab_bytes = size_t(R) * size_t(a.T) * size_t(a.m) * sizeof(double);
    int64_t blocks = capped_grid(ctx, n_groups, LORENZ_WARPS, LORENZ_FUSED_BLOCKS_PER_SM);
    const int64_t by_budget = int64_t(LORENZ_SLAB_BUDGET / (slab_bytes * LORENZ_WARPS));
    if (blocks > by_budget) blocks = by_budget < 1 ? 1 : by_budget;
    double* slab = static_cast<double*>(
        ctx_scratch(ctx, size_t(blocks) * LORENZ_WARPS * slab_bytes));
    if (!slab) return ELFI_B200_ERR_CUDA;
    sim_lorenz_fused_kernel<V><<<unsigned(blocks), LORENZ_THREADS, 0, stream>>>(a, L, R, n_groups,
                                                                                slab, S, ldS);
    return ELFI_B200_OK;
}

}  // namespace elfi

extern "C" {

int elfi_b200_sim_lorenz_f64(elfi_b200_ctx* ctx, const double* P, int64_t ldP, int64_t B,
                             int64_t n_obs, int64_t n_timestep, const double* init, double f,
                             double phi, double s_phi, double dt, uint64_t seed, uint64_t offset,
                             double* X, double* S, int64_t ldS, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || (P && init)), "sim_lorenz: NULL argument");
    ELFI_REQUIRE(n_obs >= LORENZ_M_MIN && n_obs <= LORENZ_M_MAX,
                 "sim_lorenz: %d <= n_obs <= %d, got %lld", LORENZ_M_MIN, LORENZ_M_MAX,
                 (long long)n_obs);
    ELFI_REQUIRE(n_timestep >= 2 && n_timestep <= LORENZ_T_MAX,
                 "sim_lorenz: 2 <= n_timestep <= %lld, got %lld", (long long)LORENZ_T_MAX,
                 (long long)n_timestep);
    ELFI_REQUIRE(B >= 0 && ldP >= 2, "sim_lorenz: bad shape (B=%lld ldP=%lld)", (long long)B,
                 (long long)ldP);
    ELFI_REQUIRE(S == nullptr || (ldS >= 6 && n_timestep * n_obs <= LORENZ_SUMM_MAX_TERMS),
                 "sim_lorenz: summaries need n_timestep * n_obs <= %lld and ldS >= 6",
                 (long long)LORENZ_SUMM_MAX_TERMS);
    if (B == 0 || (X == nullptr && S == nullptr)) return ELFI_B200_OK;
    LorenzSim a;
    a.P = P;
    a.ldP = ldP;
    a.B = B;
    a.m = int(n_obs);
    a.T = int(n_timestep);
    a.init = init;
    a.f = f;
    a.phi = phi;
    a.s = s_phi;
    a.dt = dt;
    a.seed = seed;
    a.offset = offset;
    const int V = lorenz_vars_per_lane(a.m);
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        return V == 1   ? launch_sim_lorenz<1>(ctx, a, X, S, ldS, stream)
               : V == 2 ? launch_sim_lorenz<2>(ctx, a, X, S, ldS, stream)
                        : launch_sim_lorenz<4>(ctx, a, X, S, ldS, stream);
    });
}

int elfi_b200_lorenz_summaries_f64(elfi_b200_ctx* ctx, const double* X, int64_t ld_row,
                                   int64_t ld_t, int64_t ld_k, int64_t B, int64_t n_timestep,
                                   int64_t n_obs, double* S, int64_t ldS, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || (X && S)), "lorenz_summaries: NULL argument");
    ELFI_REQUIRE(B >= 0 && n_obs >= ELFI_B200_LORENZ_SUMM_NOBS_MIN && n_obs <= LORENZ_M_MAX &&
                     n_timestep >= 2 && n_timestep * n_obs <= LORENZ_SUMM_MAX_TERMS && ldS >= 6,
                 "lorenz_summaries: bad shape (2 <= n_obs <= %d, 2 <= n_timestep, n_timestep * "
                 "n_obs <= %lld; n_timestep=%lld n_obs=%lld)",
                 LORENZ_M_MAX, (long long)LORENZ_SUMM_MAX_TERMS, (long long)n_timestep,
                 (long long)n_obs);
    if (B == 0) return ELFI_B200_OK;
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        const unsigned blocks = capped_grid(ctx, B, LORENZ_WARPS, 16);
        lorenz_summaries_kernel<<<blocks, LORENZ_THREADS, 0, stream>>>(
            X, ld_row, ld_t, ld_k, B, int(n_timestep), int(n_obs), S, ldS);
        return ELFI_B200_OK;
    });
}

}  // extern "C"
