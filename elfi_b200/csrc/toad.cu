// toad.cu -- the toad movement model of elfi/examples/toad.py in throughput mode: the simulator (a
// symmetric alpha-stable random walk per toad with returns to earlier refuges) and the displacement
// summaries of compute_summaries, alone or fused.
//
// Random stream (Philox4x32-10 keyed by the seed; counter (row, row >> 32, block, salt)):
//   sim_toad  row = offset + i; toad k on day d (1 <= d < n_days) uses the cell c = d * n_toads + k
//             and two blocks:
//               block (c << 1) | 0: words (x, y) -> the return uniform 1 - u01 in [0, 1),
//                                   words (z, w) -> the refuge word (z << 32) | w;
//               block (c << 1) | 1: words (x, y) -> TH = (1 - u01) * pi - pi / 2,
//                                   words (z, w) -> W = -log(u01).
// so every draw is a pure function of (seed, offset + row, d, k), whatever the thread layout; a
// returning toad does not draw block 1.  n_days * n_toads <= 2^31 keeps the block in 32 bits.
//
// Model (toad.py:16-70): X[0, k] = 0; on day d toad k returns if its uniform is < p0 and then
// takes X[j, k] with j = the high word of refuge * d (uniform in [0, d), bias below d / 2^64),
// otherwise X[d, k] = X[d - 1, k] + the levy_stable step of toad.cuh.  alpha outside (0, 2] or
// gamma < 0 (or NaN), where the reference raises, give rows of NaN.
//
// Layout: sim_toad_kernel runs one thread per (row, toad) over the days, X batch-major
// (B, n_days, n_toads) in global memory.  toad_summaries_kernel and the fused kernel run one CTA
// per row (grid-stride): the CTA writes the kept |displacements| of a lag as order-preserving keys
// (bitonic.cuh) into shared memory, compacted by warp ballots, pads them to a power of two and sorts
// them with the block-wide bitonic network; then one thread per quantile level picks and
// interpolates, and the gaps, the median and the count are written (toad.cuh).  The fused kernel
// first simulates the row into shared memory ((n_days, n_toads) doubles, 33 KB at the defaults, one
// thread per toad) and summarises it there for every requested lag: the bits of sim_toad followed
// by toad_summaries.
#include "bitonic.cuh"
#include "common.cuh"
#include "philox.cuh"
#include "toad.cuh"

namespace elfi {

constexpr uint32_t SALT_TOAD = 0x544f4144u;   // "TOAD"
constexpr int TOAD_THREADS = 256;
constexpr int TOAD_SIM_THREADS = 128;

struct ToadSim {
    const double* P;
    int64_t ldP;
    int64_t B;
    int n_toads, n_days;
    uint64_t seed, offset;
};

struct ToadSumm {
    int n_lags, n_p;
    int lags[TOAD_LAGS_MAX];
    double p[TOAD_NP_MAX];
    double thd;
};

__device__ __forceinline__ double u01_open_top(uint32_t a, uint32_t b) { return 1.0 - u01(a, b); }

// Simulates toad k of row `row` into x(d) (a callable returning a reference to day d's value).
template <class Cell>
__device__ __forceinline__ void toad_sim_one(const ToadSim& a, int64_t row, int k, const Cell& x) {
    const double alpha = a.P[row * a.ldP], gamma = a.P[row * a.ldP + 1], p0 = a.P[row * a.ldP + 2];
    if (!toad_params_ok(alpha, gamma)) {
        for (int d = 0; d < a.n_days; ++d) x(d) = NAN;
        return;
    }
    const StableRow sr = toad_stable_row(alpha, gamma);
    const Philox ph(a.seed);
    const uint64_t crow = a.offset + uint64_t(row);
    const uint32_t r0 = uint32_t(crow), r1 = uint32_t(crow >> 32);
    double cur = 0.0;
    x(0) = cur;
    for (int d = 1; d < a.n_days; ++d) {
        const uint32_t cell = uint32_t(d) * uint32_t(a.n_toads) + uint32_t(k);
        const PhiloxWords w0 = ph(r0, r1, cell << 1, SALT_TOAD);
        if (u01_open_top(w0.x, w0.y) < p0) {
            cur = x(toad_refuge_day((uint64_t(w0.z) << 32) | w0.w, d));
        } else {
            const PhiloxWords w1 = ph(r0, r1, (cell << 1) | 1u, SALT_TOAD);
            const double TH = toad_theta(u01_open_top(w1.x, w1.y));
            const double W = toad_expon(u01(w1.z, w1.w));
            cur = __dadd_rn(cur, stable_draw(sr, TH, W));
        }
        x(d) = cur;
    }
}

// The len(p) + 1 summaries of one lag of the row x(d, k), into out[0 .. n_p] (global memory).
// Every thread of the CTA calls it.  keys: TOAD_DISP_MAX words, q: TOAD_NP_MAX + 1 doubles,
// cnt: 2 ints, all shared.
template <class Get>
__device__ __forceinline__ void toad_cta_summaries(const Get& x, int n_days, int n_toads, int lag,
                                                   const ToadSumm& s, uint64_t* keys, double* q,
                                                   int* cnt, double* out) {
    const int tid = threadIdx.x, lane = tid & 31;
    const int n_rows = n_toads * (n_days - lag);
    if (tid == 0) {
        cnt[0] = 0;
        cnt[1] = 0;
    }
    __syncthreads();
    int my_ret = 0;
    for (int i0 = 0; i0 < n_rows; i0 += blockDim.x) {
        const int i = i0 + tid;
        bool kept = false;
        double ad = 0.0;
        if (i < n_rows) {
            const int t = i / n_toads, k = i - t * n_toads;
            ad = fabs(__dsub_rn(x(t + lag, k), x(t, k)));
            if (ad < s.thd)
                ++my_ret;
            else
                kept = ad == ad;
        }
        const unsigned m = __ballot_sync(0xffffffffu, kept);
        int base = 0;
        if (lane == 0 && m) base = atomicAdd(&cnt[1], __popc(m));
        base = __shfl_sync(0xffffffffu, base, 0);
        if (kept) keys[base + __popc(m & ((1u << lane) - 1u))] = key_to_u64(ad);
    }
    my_ret = __reduce_add_sync(0xffffffffu, my_ret);
    if (lane == 0 && my_ret) atomicAdd(&cnt[0], my_ret);
    __syncthreads();
    const int n = cnt[1];
    int npow2 = 1;
    while (npow2 < n) npow2 <<= 1;
    for (int i = n + tid; i < npow2; i += blockDim.x) keys[i] = ~uint64_t(0);
    __syncthreads();
    if (n > 1) bitonic_in_cta(keys, npow2);
    for (int j = tid; j <= s.n_p; j += blockDim.x) {
        double v = NAN;
        if (n > 0) {
            if (j < s.n_p) {
                const ToadPick pk = toad_quantile_pick(n, s.p[j]);
                v = gnk_lerp(u64_to_key(keys[pk.lo]), u64_to_key(keys[pk.hi]), pk.t);
            } else {
                int lo, hi;
                toad_median_picks(n, lo, hi);
                v = toad_median(u64_to_key(keys[lo]), u64_to_key(keys[hi]), n, n_rows);
            }
        }
        q[j] = v;
    }
    __syncthreads();
    for (int j = tid; j <= s.n_p; j += blockDim.x) {
        double v;
        if (j == 0)
            v = double(cnt[0]);
        else if (j == 1)
            v = q[s.n_p];
        else
            v = toad_log_gap(q[j - 2], q[j - 1]);
        out[j] = toad_nan_to_num(v);
    }
    __syncthreads();   // keys, q and cnt are reused by the next lag or row
}

// ---------------------------------------------------------------------------- kernels
// One thread per (row, toad); X (B, n_days, n_toads) C-contiguous.
__global__ void __launch_bounds__(TOAD_SIM_THREADS)
sim_toad_kernel(const ToadSim a, double* __restrict__ X) {
    const int64_t g = int64_t(blockIdx.x) * TOAD_SIM_THREADS + threadIdx.x;
    if (g >= a.B * a.n_toads) return;
    const int64_t row = g / a.n_toads;
    const int k = int(g - row * a.n_toads);
    double* xr = X + row * int64_t(a.n_days) * a.n_toads + k;
    const int nt = a.n_toads;
    toad_sim_one(a, row, k, [&](int d) -> double& { return xr[int64_t(d) * nt]; });
}

// One CTA per row, grid-stride; X[d * ld_d + k * ld_k + row * ld_b].
__global__ void __launch_bounds__(TOAD_THREADS)
toad_summaries_kernel(const double* __restrict__ X, int64_t ld_d, int64_t ld_k, int64_t ld_b,
                      int n_days, int n_toads, int64_t B, int lag, const ToadSumm s,
                      double* __restrict__ S, int64_t ldS) {
    __shared__ uint64_t keys[TOAD_DISP_MAX];
    __shared__ double q[TOAD_NP_MAX + 1];
    __shared__ int cnt[2];
    for (int64_t row = blockIdx.x; row < B; row += gridDim.x) {
        const double* xr = X + row * ld_b;
        toad_cta_summaries([&](int d, int k) { return xr[d * ld_d + k * ld_k]; }, n_days, n_toads,
                           lag, s, keys, q, cnt, S + row * ldS);
    }
}

// Fused: one CTA per row, grid-stride; the trajectory lives in dynamic shared memory.
__global__ void __launch_bounds__(TOAD_THREADS)
sim_toad_fused_kernel(const ToadSim a, const ToadSumm s, double* __restrict__ S, int64_t ldS) {
    __shared__ uint64_t keys[TOAD_DISP_MAX];
    __shared__ double q[TOAD_NP_MAX + 1];
    __shared__ int cnt[2];
    extern __shared__ double traj[];
    const int nt = a.n_toads;
    const int w = s.n_p + 1;
    for (int64_t row = blockIdx.x; row < a.B; row += gridDim.x) {
        for (int k = threadIdx.x; k < nt; k += blockDim.x)
            toad_sim_one(a, row, k, [&](int d) -> double& { return traj[d * nt + k]; });
        __syncthreads();
        for (int l = 0; l < s.n_lags; ++l)
            toad_cta_summaries([&](int d, int k) { return traj[d * nt + k]; }, a.n_days, nt,
                               s.lags[l], s, keys, q, cnt, S + row * ldS + l * w);
    }
}

static int toad_summ_args(ToadSumm& s, int64_t n_lags, const int64_t* lags, int64_t n_p,
                          const double* p, double thd) {
    s.n_lags = int(n_lags);
    s.n_p = int(n_p);
    for (int l = 0; l < TOAD_LAGS_MAX; ++l) s.lags[l] = l < n_lags ? int(lags[l]) : 0;
    for (int j = 0; j < TOAD_NP_MAX; ++j) s.p[j] = j < n_p ? p[j] : 0.0;
    s.thd = thd;
    return 0;
}

}  // namespace elfi

extern "C" {

int elfi_b200_sim_toad_f64(elfi_b200_ctx* ctx, const double* P, int64_t ldP, int64_t B,
                           int64_t n_toads, int64_t n_days, uint64_t seed, uint64_t offset,
                           double* X, int64_t n_lags, const int64_t* lags, int64_t n_p,
                           const double* p, double thd, double* S, int64_t ldS, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || P), "sim_toad: NULL argument");
    ELFI_REQUIRE(B >= 0 && ldP >= 3 && n_toads >= 1 && n_days >= 1 &&
                     n_days * n_toads <= TOAD_CELLS_MAX,
                 "sim_toad: bad shape (B=%lld ldP=%lld n_toads=%lld n_days=%lld; n_days * n_toads "
                 "<= 2^31)", (long long)B, (long long)ldP, (long long)n_toads, (long long)n_days);
    if (S) {
        ELFI_REQUIRE(lags && p && n_lags >= 1 && n_lags <= TOAD_LAGS_MAX && n_p >= 1 &&
                         n_p <= TOAD_NP_MAX && ldS >= n_lags * (n_p + 1),
                     "sim_toad: summaries need 1 <= n_lags <= %d, 1 <= n_p <= %d and ldS >= "
                     "n_lags * (n_p + 1)", TOAD_LAGS_MAX, TOAD_NP_MAX);
        ELFI_REQUIRE(n_toads * (n_days - 1) <= TOAD_DISP_MAX,
                     "sim_toad: summaries need n_toads * (n_days - 1) <= %d", TOAD_DISP_MAX);
        for (int64_t l = 0; l < n_lags; ++l)
            ELFI_REQUIRE(lags[l] >= 1 && lags[l] < n_days, "sim_toad: lag %lld outside [1, n_days)",
                         (long long)lags[l]);
    }
    if (B == 0 || (X == nullptr && S == nullptr)) return ELFI_B200_OK;
    ToadSim a;
    a.P = P;
    a.ldP = ldP;
    a.B = B;
    a.n_toads = int(n_toads);
    a.n_days = int(n_days);
    a.seed = seed;
    a.offset = offset;
    ToadSumm s;
    if (S) toad_summ_args(s, n_lags, lags, n_p, p, thd);
    const unsigned grid = capped_grid(ctx, B, 1, 8);   // a CTA per row, at most 8 per SM
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        if (X) {
            const int64_t blocks = (B * n_toads + TOAD_SIM_THREADS - 1) / TOAD_SIM_THREADS;
            ELFI_REQUIRE(blocks < (int64_t(1) << 31), "sim_toad: B * n_toads too large");
            sim_toad_kernel<<<unsigned(blocks), TOAD_SIM_THREADS, 0, stream>>>(a, X);
            ELFI_CUDA_OK(cudaGetLastError());
            if (S) {
                const int64_t nt = n_days * n_toads;
                for (int64_t l = 0; l < n_lags; ++l) {
                    toad_summaries_kernel<<<grid, TOAD_THREADS, 0, stream>>>(
                        X, n_toads, 1, nt, int(n_days), int(n_toads), B, int(lags[l]), s,
                        S + l * (n_p + 1), ldS);
                    ELFI_CUDA_OK(cudaGetLastError());
                }
            }
            return ELFI_B200_OK;
        }
        const size_t smem = size_t(n_days * n_toads) * sizeof(double);
        ELFI_CUDA_OK(cudaFuncSetAttribute(sim_toad_fused_kernel,
                                          cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
        sim_toad_fused_kernel<<<grid, TOAD_THREADS, smem, stream>>>(a, s, S, ldS);
        return ELFI_B200_OK;
    });
}

int elfi_b200_toad_summaries_f64(elfi_b200_ctx* ctx, const double* X, int64_t ld_day,
                                 int64_t ld_toad, int64_t ld_row, int64_t n_days, int64_t n_toads,
                                 int64_t B, int64_t lag, int64_t n_p, const double* p, double thd,
                                 double* S, int64_t ldS, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && p && (B == 0 || (X && S)), "toad_summaries: NULL argument");
    ELFI_REQUIRE(B >= 0 && n_toads >= 1 && lag >= 1 && lag < n_days &&
                     n_toads * (n_days - lag) <= TOAD_DISP_MAX && n_p >= 1 && n_p <= TOAD_NP_MAX &&
                     ldS >= n_p + 1,
                 "toad_summaries: bad shape (1 <= lag < n_days, n_toads * (n_days - lag) <= %d, "
                 "1 <= n_p <= %d; n_days=%lld n_toads=%lld lag=%lld n_p=%lld)", TOAD_DISP_MAX,
                 TOAD_NP_MAX, (long long)n_days, (long long)n_toads, (long long)lag,
                 (long long)n_p);
    if (B == 0) return ELFI_B200_OK;
    ToadSumm s;
    toad_summ_args(s, 1, &lag, n_p, p, thd);
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        toad_summaries_kernel<<<capped_grid(ctx, B, 1, 8), TOAD_THREADS, 0, stream>>>(
            X, ld_day, ld_toad, ld_row, int(n_days), int(n_toads), B, int(lag), s, S, ldS);
        return ELFI_B200_OK;
    });
}

}  // extern "C"
