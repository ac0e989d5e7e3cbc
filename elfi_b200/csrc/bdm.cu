// bdm.cu -- the birth-death-mutation model of elfi/examples/bdm.py (the reference's external
// executable elfi/examples/cpp/bdm.cpp, --mode 1) in throughput mode: the simulator with the
// summaries T1 and T2 fused, and the summaries of written counts.  bdm.cuh has the arithmetic.
//
// Random streams (Philox4x32-10 keyed by the seed; counter (row, row >> 32, k, SALT_BDM)), with
// row = offset + i: event k (0 <= k < max_events) draws u = 1 - u01(x, y) and v = 1 - u01(z, w),
// both in [0, 1), so every row is a pure function of (seed, offset + i), whatever lane or launch
// ran it.
//
// Layout: the simulator is persistent (grid = SMs x the resident blocks per SM).  A lane runs one
// row at a time; its N counts live in shared memory as uint16, interleaved across the CTA's lanes
// (count j of lane l at [j * blockDim.x + l]) so that lanes scanning the same j read neighbouring
// halves of one bank word.  Rows are handed out by a per-launch counter: whenever lanes of a warp
// have finished their rows, one warp-aggregated atomicAdd claims as many new row indices and the
// idle lanes take them, so a warp is not held up by its slowest row (event counts differ by orders
// of magnitude across the prior).  The CTA has 32 to 256 lanes, as many as keep its counts within
// 48 KB (eight warps up to N = 96, one warp from N = 385 up, 64 KB for one warp at N = 1024).
//
// A row whose rates bdm_init refuses gets counts of -1, NaN summaries and n_events = -1; a row
// still running after max_events events gets counts of -1, NaN summaries and n_events =
// max_events.
//
// bdm_summaries_kernel: one thread per row, reading X[row * ld_row + j * ld_col] (int16); a row
// with a negative count (the mark of an invalid or capped row) gets NaN summaries.
#include "bdm.cuh"
#include "common.cuh"
#include "philox.cuh"

namespace elfi {

constexpr uint32_t SALT_BDM = 0x42444d31u;   // "BDM1"
constexpr int BDM_THREADS_MAX = 256;
constexpr int BDM_SMEM_TARGET = 48 * 1024;
constexpr int BDM_SUMM_THREADS = 128;

struct BdmSim {
    const double* P;        // (B, 3; ldP): alpha, delta, tau
    int64_t ldP;
    int64_t B;
    int N;
    double n_t2;            // T2's argument
    uint32_t max_events;
    uint64_t seed, offset;
    int16_t* X;             // (B, N; ldX) or NULL
    int64_t ldX;
    double* S;              // (B, 2; ldS) or NULL
    int64_t ldS;
    int64_t* n_events;      // (B,)
    unsigned long long* next_row;   // per-launch row counter, starts at 0
};

// Writes a finished row: its counts and summaries (ok), or -1 counts and NaN summaries.
__device__ __forceinline__ void bdm_write(const BdmSim& a, int64_t row, const uint16_t* c,
                                          int stride, bool ok, int64_t n_events) {
    if (a.X) {
        int16_t* x = a.X + row * a.ldX;
        for (int j = 0; j < a.N; ++j) x[j] = ok ? int16_t(c[j * stride]) : int16_t(-1);
    }
    if (a.S) {
        double* s = a.S + row * a.ldS;
        if (ok) {
            bdm_summaries(a.N, a.n_t2, [&](int j) { return c[j * stride]; }, s);
        } else {
            s[0] = NAN;
            s[1] = NAN;
        }
    }
    a.n_events[row] = n_events;
}

// Runs one event of the lane's row.  Returns false when the row is finished (and written).
__device__ __forceinline__ bool bdm_lane_step(const BdmSim& a, const Philox& ph, int64_t row,
                                              BdmState& s, uint16_t* c, int stride) {
    if (!bdm_running(s)) {
        bdm_finish(s, c, stride);
        bdm_write(a, row, c, stride, true, s.k);
        return false;
    }
    if (s.k >= a.max_events) {
        bdm_write(a, row, c, stride, false, s.k);
        return false;
    }
    const uint64_t crow = a.offset + uint64_t(row);
    const PhiloxWords w = ph(uint32_t(crow), uint32_t(crow >> 32), s.k, SALT_BDM);
    bdm_step(s, 1.0 - u01(w.x, w.y), 1.0 - u01(w.z, w.w), c, stride);
    return true;
}

__global__ void __launch_bounds__(BDM_THREADS_MAX)
sim_bdm_kernel(const BdmSim a) {
    extern __shared__ uint16_t bdm_counts[];
    const int stride = blockDim.x;
    uint16_t* c = bdm_counts + threadIdx.x;
    const int lane = threadIdx.x & 31;
    const Philox ph(a.seed);
    BdmState s;
    int64_t row = -1;
    for (;;) {
        // lanes without a row claim new ones, one atomic per warp
        const bool idle = row < 0;
        const unsigned want = __ballot_sync(0xffffffffu, idle);
        if (want) {
            unsigned long long base = 0;
            const int leader = __ffs(want) - 1;
            if (lane == leader) base = atomicAdd(a.next_row, (unsigned long long)__popc(want));
            base = __shfl_sync(0xffffffffu, base, leader);
            if (idle) {
                const unsigned long long r = base + __popc(want & ((1u << lane) - 1u));
                row = r < (unsigned long long)a.B ? int64_t(r) : a.B;
                if (row < a.B) {
                    const double* p = a.P + row * a.ldP;
                    if (!bdm_init(s, p[0], p[1], p[2], a.N, c, stride)) {
                        bdm_write(a, row, c, stride, false, -1);
                        row = -1;
                    }
                }
            }
        }
        if (__all_sync(0xffffffffu, row >= a.B)) break;
        // run events until some lane of the warp has finished its row
        while (!__any_sync(0xffffffffu, row < 0)) {
            const bool live = row < a.B;
            if (__all_sync(0xffffffffu, !live)) break;
            if (live && !bdm_lane_step(a, ph, row, s, c, stride)) row = -1;
        }
    }
}

__global__ void __launch_bounds__(BDM_SUMM_THREADS)
bdm_summaries_kernel(const int16_t* __restrict__ X, int64_t ld_row, int64_t ld_col, int64_t B,
                     int N, double n, double* __restrict__ S, int64_t ldS) {
    const int64_t stride = int64_t(gridDim.x) * blockDim.x;
    for (int64_t row = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; row < B; row += stride) {
        const int16_t* x = X + row * ld_row;
        double* s = S + row * ldS;
        bool ok = true;
        for (int j = 0; j < N; ++j) ok = ok && x[j * ld_col] >= 0;
        if (ok) {
            bdm_summaries(N, n, [&](int j) { return x[j * ld_col]; }, s);
        } else {
            s[0] = NAN;
            s[1] = NAN;
        }
    }
}

// lanes per CTA for N counts per lane: a multiple of 32 whose counts fit BDM_SMEM_TARGET
inline int bdm_threads(int N) {
    int warps = BDM_SMEM_TARGET / (32 * 2 * N);
    if (warps < 1) warps = 1;
    if (warps > BDM_THREADS_MAX / 32) warps = BDM_THREADS_MAX / 32;
    return 32 * warps;
}

}  // namespace elfi

extern "C" {

int elfi_b200_sim_bdm_f64(elfi_b200_ctx* ctx, const double* P, int64_t ldP, int64_t B, int64_t N,
                          double n_t2, int64_t max_events, uint64_t seed, uint64_t offset,
                          int16_t* X, int64_t ldX, double* S, int64_t ldS, int64_t* n_events,
                          void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || (P && n_events)), "sim_bdm: NULL argument");
    ELFI_REQUIRE(B >= 0 && B <= ELFI_B200_BDM_BATCH_MAX && ldP >= 3 && N >= 1 && N <= BDM_N_MAX &&
                     (!X || ldX >= N) && (!S || ldS >= BDM_NSUMM),
                 "sim_bdm: bad shape (1 <= N <= %d, B < 2^31, ldP >= 3, ldX >= N, ldS >= 2; "
                 "B=%lld N=%lld ldP=%lld ldX=%lld ldS=%lld)", BDM_N_MAX, (long long)B,
                 (long long)N, (long long)ldP, (long long)ldX, (long long)ldS);
    ELFI_REQUIRE(max_events >= 1 && max_events <= ELFI_B200_BDM_MAX_EVENTS_LIMIT,
                 "sim_bdm: 1 <= max_events <= 2^32 - 1 (the event is one Philox word), got %lld",
                 (long long)max_events);
    if (B == 0) return ELFI_B200_OK;
    BdmSim a;
    a.P = P;
    a.ldP = ldP;
    a.B = B;
    a.N = int(N);
    a.n_t2 = n_t2;
    a.max_events = uint32_t(max_events);
    a.seed = seed;
    a.offset = offset;
    a.X = X;
    a.ldX = ldX;
    a.S = S;
    a.ldS = ldS;
    a.n_events = n_events;
    const int threads = bdm_threads(int(N));
    const size_t smem = size_t(2) * size_t(N) * size_t(threads);
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        auto* counter = static_cast<unsigned long long*>(ctx_scratch(ctx, 256));
        if (!counter) return ELFI_B200_ERR_CUDA;
        ELFI_CUDA_OK(cudaMemsetAsync(counter, 0, sizeof(unsigned long long), stream));
        a.next_row = counter;
        ELFI_CUDA_OK(cudaFuncSetAttribute(sim_bdm_kernel,
                                          cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
        int per_sm = 0;
        ELFI_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, sim_bdm_kernel,
                                                                   threads, smem));
        if (per_sm < 1) per_sm = 1;
        sim_bdm_kernel<<<capped_grid(ctx, B, threads, per_sm), threads, smem, stream>>>(a);
        return ELFI_B200_OK;
    });
}

int elfi_b200_bdm_summaries_f64(elfi_b200_ctx* ctx, const int16_t* X, int64_t ld_row,
                                int64_t ld_col, int64_t B, int64_t N, double n, double* S,
                                int64_t ldS, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || (X && S)), "bdm_summaries: NULL argument");
    ELFI_REQUIRE(B >= 0 && N >= 1 && N <= BDM_N_MAX && ldS >= BDM_NSUMM,
                 "bdm_summaries: bad shape (1 <= N <= %d, ldS >= 2; N=%lld ldS=%lld)", BDM_N_MAX,
                 (long long)N, (long long)ldS);
    if (B == 0) return ELFI_B200_OK;
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        const unsigned blocks = capped_grid(ctx, B, BDM_SUMM_THREADS, 32);
        bdm_summaries_kernel<<<blocks, BDM_SUMM_THREADS, 0, stream>>>(X, ld_row, ld_col, B, int(N),
                                                                      n, S, ldS);
        return ELFI_B200_OK;
    });
}

}  // extern "C"
