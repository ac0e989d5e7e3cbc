// lotka_volterra.cu -- the stochastic Lotka-Volterra model of elfi/examples/lotka_volterra.py in
// throughput mode: Gillespie's direct method per row, observed at n_obs times, and the nine
// summaries of the observations (a second kernel).
//
// Random streams (Philox4x32-10 keyed by the seed; counter (row, row >> 32, block, salt)), with
// row = offset + i:
//   event k (0 <= k < max_events)  block k, salt SALT_LV: E = -log(u01(x, y)), the reaction
//                                  uniform 1 - u01(z, w) in [0, 1)
//   observation j (1 <= j < n_obs) block j, salt SALT_LV_NOISE: the Box-Muller pair
//                                  (boxmuller.cuh), prey noise sigma n0, predator noise sigma n1
// so every value is a pure function of (seed, offset + row, k or j), whatever lane or launch ran
// the row.  The noise blocks are drawn only when sigma != 0 (sigma * n is then 0 anyway).
//
// Layout: the simulator is persistent (grid = SMs x the resident blocks per SM).  A lane runs one
// row at a time, keeping (t, X, Y) in registers, and emits observation j (both species) when an
// event reaches t_out[j] (staged in shared memory).  Rows are handed out by a per-launch counter:
// whenever lanes of a warp have finished their rows, one warp-aggregated atomicAdd claims as many
// new row indices and the idle lanes take them, so a warp is not held up by its slowest row.
// A row runs at most max_events events; one that has not reached time_end by then, whose
// parameters the reference rejects (a negative or NaN rate or sigma, initial counts floor(prey0)
// or floor(predator0) outside [0, 2^31)) or whose total hazard turns negative or NaN gets NaN
// observations.  n_events is the number of events the row ran (max_events for a capped row).
//
// lv_summaries_kernel: one thread per row, reading X[row * ld_b + t * ld_t + s * ld_s]
// (lotka_volterra.cuh has the arithmetic).
#include "boxmuller.cuh"
#include "common.cuh"
#include "lotka_volterra.cuh"
#include "philox.cuh"

namespace elfi {

constexpr uint32_t SALT_LV = 0x4c4f5456u;         // "LOTV"
constexpr uint32_t SALT_LV_NOISE = 0x4c564e4fu;   // "LVNO"
constexpr int LV_THREADS = 256;
constexpr int LV_SUMM_THREADS = 128;

struct LvSim {
    const double* P;        // (B, 6; ldP): r1, r2, r3, prey0, predator0, sigma
    int64_t ldP;
    int64_t B;
    const double* t_out;    // (n_obs,), t_out[0] = 0 and t_out[n_obs - 1] = time_end
    int n_obs;
    double time_end;
    uint32_t max_events;
    uint64_t seed, offset;
    double* X;              // (B, n_obs, 2)
    int64_t* n_events;      // (B,)
    unsigned long long* next_row;   // per-launch row counter, starts at 0
};

__device__ __forceinline__ void lv_nan_row(const LvSim& a, int64_t row) {
    double* x = a.X + row * int64_t(a.n_obs) * 2;
    for (int i = 0; i < 2 * a.n_obs; ++i) x[i] = NAN;
}

// One lane's row: its index (-1: claim one, >= B: no rows left) and its state.
struct LvLane {
    int64_t row;
    LvState s;
};

// Starts the lane's row and writes observation 0.  Returns false (the row is finished, with NaN
// observations) when the parameters are rejected.
__device__ __forceinline__ bool lv_start(const LvSim& a, LvLane& l) {
    if (!lv_init(l.s, a.P + l.row * a.ldP)) {
        lv_nan_row(a, l.row);
        a.n_events[l.row] = 0;
        return false;
    }
    double* x = a.X + l.row * int64_t(a.n_obs) * 2;
    x[0] = l.s.X;
    x[1] = l.s.Y;
    return true;
}

// Runs one event of the lane's row.  Returns false when the row is finished (and written).
__device__ __forceinline__ bool lv_step(const LvSim& a, const Philox& ph, const double* t_out,
                                        LvLane& l) {
    const uint64_t crow = a.offset + uint64_t(l.row);
    const uint32_t c0 = uint32_t(crow), c1 = uint32_t(crow >> 32);
    bool ok = lv_running(l.s, a.time_end, a.max_events);
    if (ok) {
        const PhiloxWords w = ph(c0, c1, l.s.k, SALT_LV);
        double* x = a.X + l.row * int64_t(a.n_obs) * 2;
        ok = lv_advance(
            l.s, -log(u01(w.x, w.y)), 1.0 - u01(w.z, w.w), t_out, a.n_obs, a.time_end,
            [&](int j, double& n0, double& n1) {
                normal2(ph(c0, c1, uint32_t(j), SALT_LV_NOISE), n0, n1);
            },
            [&](int j, double prey, double pred) {
                x[2 * j] = prey;
                x[2 * j + 1] = pred;
            });
        if (ok) return true;
    } else if (lv_complete(l.s, a.time_end, a.n_obs)) {
        a.n_events[l.row] = l.s.k;
        return false;
    }
    // capped, a NaN time or an invalid hazard
    lv_nan_row(a, l.row);
    a.n_events[l.row] = l.s.k;
    return false;
}

__global__ void __launch_bounds__(LV_THREADS)
sim_lv_kernel(const LvSim a) {
    __shared__ double t_out[LV_NOBS_MAX];
    for (int i = threadIdx.x; i < a.n_obs; i += blockDim.x) t_out[i] = a.t_out[i];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const Philox ph(a.seed);
    LvLane l;
    l.row = -1;
    for (;;) {
        // lanes without a row claim new ones, one atomic per warp
        const bool idle = l.row < 0;
        const unsigned want = __ballot_sync(0xffffffffu, idle);
        if (want) {
            unsigned long long base = 0;
            const int leader = __ffs(want) - 1;
            if (lane == leader) base = atomicAdd(a.next_row, (unsigned long long)__popc(want));
            base = __shfl_sync(0xffffffffu, base, leader);
            if (idle) {
                const unsigned long long r = base + __popc(want & ((1u << lane) - 1u));
                l.row = r < (unsigned long long)a.B ? int64_t(r) : a.B;
                if (l.row < a.B && !lv_start(a, l)) l.row = -1;
            }
        }
        if (__all_sync(0xffffffffu, l.row >= a.B)) break;
        // run events until some lane of the warp has finished its row
        while (!__any_sync(0xffffffffu, l.row < 0)) {
            const bool live = l.row < a.B;
            if (__all_sync(0xffffffffu, !live)) break;
            if (live && !lv_step(a, ph, t_out, l)) l.row = -1;
        }
    }
}

__global__ void __launch_bounds__(LV_SUMM_THREADS)
lv_summaries_kernel(const double* __restrict__ X, int64_t ld_b, int64_t ld_t, int64_t ld_s,
                    int64_t B, int n, double* __restrict__ S, int64_t ldS) {
    const int64_t stride = int64_t(gridDim.x) * blockDim.x;
    for (int64_t row = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; row < B; row += stride) {
        const double* x = X + row * ld_b;
        double out[LV_NSUMM];
        lv_summaries(n, [&](int i, int sp) { return x[i * ld_t + sp * ld_s]; }, out);
        for (int c = 0; c < LV_NSUMM; ++c) S[row * ldS + c] = out[c];
    }
}

}  // namespace elfi

extern "C" {

int elfi_b200_sim_lotka_volterra_f64(elfi_b200_ctx* ctx, const double* P, int64_t ldP, int64_t B,
                                     const double* t_out, int64_t n_obs, double time_end,
                                     int64_t max_events, uint64_t seed, uint64_t offset,
                                     double* X, int64_t* n_events, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || (P && t_out && X && n_events)),
                 "sim_lotka_volterra: NULL argument");
    ELFI_REQUIRE(B >= 0 && ldP >= 6 && n_obs >= 1 && n_obs <= LV_NOBS_MAX,
                 "sim_lotka_volterra: bad shape (1 <= n_obs <= %d, ldP >= 6; B=%lld n_obs=%lld "
                 "ldP=%lld)", LV_NOBS_MAX, (long long)B, (long long)n_obs, (long long)ldP);
    ELFI_REQUIRE(time_end > 0.0 && time_end < INFINITY,
                 "sim_lotka_volterra: time_end must be finite and > 0");
    ELFI_REQUIRE(max_events >= 1 && max_events <= ELFI_B200_LV_MAX_EVENTS_LIMIT,
                 "sim_lotka_volterra: 1 <= max_events <= 2^32 - 1 (the event is one Philox word), "
                 "got %lld", (long long)max_events);
    if (B == 0) return ELFI_B200_OK;
    LvSim a;
    a.P = P;
    a.ldP = ldP;
    a.B = B;
    a.t_out = t_out;
    a.n_obs = int(n_obs);
    a.time_end = time_end;
    a.max_events = uint32_t(max_events);
    a.seed = seed;
    a.offset = offset;
    a.X = X;
    a.n_events = n_events;
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        auto* counter = static_cast<unsigned long long*>(ctx_scratch(ctx, 256));
        if (!counter) return ELFI_B200_ERR_CUDA;
        ELFI_CUDA_OK(cudaMemsetAsync(counter, 0, sizeof(unsigned long long), stream));
        a.next_row = counter;
        int per_sm = 0;
        ELFI_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, sim_lv_kernel,
                                                                   LV_THREADS, 0));
        if (per_sm < 1) per_sm = 1;
        sim_lv_kernel<<<capped_grid(ctx, B, LV_THREADS, per_sm), LV_THREADS, 0, stream>>>(a);
        return ELFI_B200_OK;
    });
}

int elfi_b200_lv_summaries_f64(elfi_b200_ctx* ctx, const double* X, int64_t ld_row, int64_t ld_obs,
                               int64_t ld_species, int64_t B, int64_t n_obs, double* S,
                               int64_t ldS, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || (X && S)), "lv_summaries: NULL argument");
    ELFI_REQUIRE(B >= 0 && n_obs >= LV_SUMM_NOBS_MIN && n_obs <= LV_SUMM_NOBS_MAX &&
                     ldS >= LV_NSUMM,
                 "lv_summaries: bad shape (%d <= n_obs <= %d, ldS >= %d; n_obs=%lld ldS=%lld)",
                 LV_SUMM_NOBS_MIN, LV_SUMM_NOBS_MAX, LV_NSUMM, (long long)n_obs, (long long)ldS);
    if (B == 0) return ELFI_B200_OK;
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        const unsigned blocks = capped_grid(ctx, B, LV_SUMM_THREADS, 32);
        lv_summaries_kernel<<<blocks, LV_SUMM_THREADS, 0, stream>>>(
            X, ld_row, ld_obs, ld_species, B, int(n_obs), S, ldS);
        return ELFI_B200_OK;
    });
}

}  // extern "C"
