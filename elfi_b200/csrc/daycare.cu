// daycare.cu -- the day care model of elfi/examples/daycare.py in throughput mode: the simulator
// (Gillespie's direct method in every DCC of a row, with the four summaries fused), the summaries
// of written data, and the sorted-L1 distance.  daycare.cuh has the arithmetic.
//
// Law: within a row the DCCs step in lock-step.  If DCC c needs k_c transitions to pass time_end,
// every DCC of the row takes K = max_c k_c transitions (the crossing one included), which is the
// reference's law at batch_size = 1.  The reference steps its whole batch in lock-step instead, so
// its law depends on the batch; a row here is a pure function of (seed, row).
//
// Random streams (Philox4x32-10 keyed by the seed; counter (row, row >> 32, k, SALT_DAYCARE + c)),
// row = offset + i: transition k (0-based) of DCC c draws E = -log(u01(x, y)) and the uniform
// 1 - u01(z, w) in [0, 1).
//
// Layout: one warp per row, one lane per DCC (n_dcc <= 32), one CTA per row.  Each lane keeps its
// DCC's state in shared memory, interleaved across the lanes (element i of lane l at [i * 32 + l]),
// and every lane steps until no lane of the row is short of time_end, so K is the loop count.  A
// row that dc_row_ok refuses (t1, t2 or t3 negative, NaN or infinite, or an expected number of
// transitions that could reach the event word), a launch whose freq has a negative or non-finite
// value, and a row in which some transition finds no positive weight (a NaN waiting time) get NaN
// summaries, all-zero data and K = -1; a row that reaches 2^32 - 1 transitions gets NaN summaries
// and K = 2^32 - 1.
//
// daycare_summaries_kernel: one thread per (row, DCC), reading X[b * ld_b + c * ld_c + i * ld_i +
// s * ld_s] (uint8, nonzero = carrier) into strain masks and calling the same dc_summaries.
// daycare_distance_kernel: one thread per row.
#include "common.cuh"
#include "daycare.cuh"
#include "philox.cuh"

namespace elfi {

constexpr uint32_t SALT_DAYCARE = 0x44434300u;   // "DCC" + the DCC index in the low byte
constexpr int DC_DIST_THREADS = 128;
constexpr int DC_SUMM_THREADS = 128;

struct DcSim {
    const double* P;      // (B, 3; ldP): t1, t2, t3
    int64_t ldP, B;
    int n_dcc, n_ind, n_strains, n_obs;
    const double* f;      // (n_strains) device
    int64_t L;
    double time_end;
    uint64_t seed, offset;
    double* S;            // (B, 4 n_dcc; ldS) or NULL
    int64_t ldS;
    uint8_t* X;           // (B, n_dcc, n_obs, n_strains) or NULL
    int64_t* K;           // (B,)
};

__global__ void __launch_bounds__(32)
sim_daycare_kernel(const DcSim a) {
    extern __shared__ uint64_t smem[];
    __shared__ double f[DC_STRAINS_MAX];
    __shared__ int64_t Lk[DC_STRAINS_MAX + 1];
    const int lane = threadIdx.x;
    const int64_t row = blockIdx.x;
    for (int s = lane; s < a.n_strains; s += 32) f[s] = a.f[s];
    for (int k = 1 + lane; k <= a.n_strains; k += 32) Lk[k] = a.L / k;
    __syncwarp();
    const double* prm = a.P + row * a.ldP;
    DcParams p;
    p.t1 = prm[0];
    p.t2 = prm[1];
    p.t3 = prm[2];
    p.nf = 1.0 / double(a.n_ind - 1);
    p.Ld = double(a.L);
    p.f = f;
    p.Lk = Lk;
    p.n_ind = a.n_ind;
    p.n_strains = a.n_strains;
    DcState st;
    st.mask = smem + lane;
    st.num = reinterpret_cast<int64_t*>(smem + 32 * a.n_ind) + lane;
    st.cnt = reinterpret_cast<int32_t*>(smem + 32 * (a.n_ind + a.n_strains)) + lane;
    st.stride = 32;
    const bool active = lane < a.n_dcc;
    bool f_ok = true;
    double f_max = 0.0;
    for (int s = 0; s < a.n_strains; ++s) {
        f_ok = f_ok && f[s] >= 0.0 && f[s] < INFINITY;
        f_max = fmax(f_max, f[s]);
    }
    bool valid = f_ok && dc_row_ok(p.t1, p.t2, p.t3, f_max, a.n_ind, a.n_strains, a.time_end);
    if (active) dc_clear(st, p);
    const uint64_t crow = a.offset + uint64_t(row);
    const uint32_t c0 = uint32_t(crow), c1 = uint32_t(crow >> 32);
    const Philox ph(a.seed);
    double t = 0.0;
    uint32_t k = 0;
    bool capped = false;
    if (valid) {
        while (__any_sync(0xffffffffu, active && t < a.time_end)) {
            if (k == 0xffffffffu) {
                capped = true;
                break;
            }
            if (active) {
                const PhiloxWords w = ph(c0, c1, k, SALT_DAYCARE + uint32_t(lane));
                t = leaf_add(t, dc_step(p, st, -log(u01(w.x, w.y)), 1.0 - u01(w.z, w.w)));
            }
            ++k;
        }
        // a NaN time: some transition of the row found no positive weight
        if (__any_sync(0xffffffffu, active && !(t >= 0.0))) valid = false;
    }
    if (lane == 0) a.K[row] = !valid ? -1 : int64_t(k);
    if (!active) return;
    if (a.S) {
        double* out = a.S + row * a.ldS + lane;
        if (!valid || capped) {
            for (int j = 0; j < DC_NSUMM; ++j) out[j * a.n_dcc] = NAN;
        } else {
            dc_summaries(a.n_obs, a.n_strains, [&](int i) { return st.mask[i * 32]; }, out,
                         a.n_dcc);
        }
    }
    if (a.X) {
        uint8_t* x = a.X + (row * a.n_dcc + lane) * int64_t(a.n_obs) * a.n_strains;
        for (int i = 0; i < a.n_obs; ++i) {
            const uint64_t m = valid ? st.mask[i * 32] : 0;
            for (int s = 0; s < a.n_strains; ++s) x[i * a.n_strains + s] = uint8_t((m >> s) & 1);
        }
    }
}

__global__ void __launch_bounds__(DC_SUMM_THREADS)
daycare_summaries_kernel(const uint8_t* __restrict__ X, int64_t ld_b, int64_t ld_c, int64_t ld_i,
                         int64_t ld_s, int64_t B, int n_dcc, int n_obs, int n_strains,
                         double* __restrict__ S, int64_t ldS) {
    const int64_t n = B * n_dcc;
    const int64_t stride = int64_t(gridDim.x) * blockDim.x;
    for (int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; j < n; j += stride) {
        const int64_t b = j / n_dcc;
        const int c = int(j - b * n_dcc);
        const uint8_t* x = X + b * ld_b + c * ld_c;
        dc_summaries(n_obs, n_strains, [&](int i) {
            uint64_t m = 0;
            for (int s = 0; s < n_strains; ++s)
                m |= uint64_t(x[i * ld_i + s * ld_s] != 0) << s;
            return m;
        }, S + b * ldS + c, n_dcc);
    }
}

__global__ void __launch_bounds__(DC_DIST_THREADS)
daycare_distance_kernel(const double* __restrict__ S, int64_t ldS, int64_t B, int n_ss, int n_dcc,
                        const double* __restrict__ obs_max, const double* __restrict__ y,
                        double* __restrict__ d) {
    const int64_t stride = int64_t(gridDim.x) * blockDim.x;
    for (int64_t b = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; b < B; b += stride) {
        const double* s = S + b * ldS;
        d[b] = dc_distance(n_ss, n_dcc, [&](int k, int c) { return s[k * n_dcc + c]; }, obs_max, y,
                           B == 1);
    }
}

}  // namespace elfi

extern "C" {

int elfi_b200_sim_daycare_f64(elfi_b200_ctx* ctx, const double* P, int64_t ldP, int64_t B,
                              int64_t n_dcc, int64_t n_ind, int64_t n_strains,
                              const double* freq, int64_t n_obs, double time_end, uint64_t seed,
                              uint64_t offset, double* S, int64_t ldS, uint8_t* X, int64_t* K,
                              void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || (P && freq && K)), "sim_daycare: NULL argument");
    ELFI_REQUIRE(B >= 0 && B <= ELFI_B200_DC_BATCH_MAX && ldP >= 3 && n_dcc >= 1 &&
                     n_dcc <= DC_DCC_MAX && n_ind >= 2 && n_ind <= DC_IND_MAX && n_strains >= 1 &&
                     n_strains <= DC_STRAINS_MAX && n_obs >= 1 && n_obs <= n_ind &&
                     (!S || ldS >= DC_NSUMM * n_dcc),
                 "sim_daycare: bad shape (1 <= n_dcc <= %d, 2 <= n_ind <= %d, 1 <= n_strains <= "
                 "%d, 1 <= n_obs <= n_ind, B < 2^31; B=%lld n_dcc=%lld n_ind=%lld n_strains=%lld "
                 "n_obs=%lld)", DC_DCC_MAX, DC_IND_MAX, DC_STRAINS_MAX, (long long)B,
                 (long long)n_dcc, (long long)n_ind, (long long)n_strains, (long long)n_obs);
    ELFI_REQUIRE(time_end > 0.0 && time_end < INFINITY,
                 "sim_daycare: time_end must be finite and > 0");
    if (B == 0) return ELFI_B200_OK;
    DcSim a;
    a.P = P;
    a.ldP = ldP;
    a.B = B;
    a.n_dcc = int(n_dcc);
    a.n_ind = int(n_ind);
    a.n_strains = int(n_strains);
    a.n_obs = int(n_obs);
    a.f = freq;
    a.L = dc_lcm(int(n_strains));
    a.time_end = time_end;
    a.seed = seed;
    a.offset = offset;
    a.S = S;
    a.ldS = ldS;
    a.X = X;
    a.K = K;
    const size_t smem = 32 * (8 * size_t(n_ind) + 12 * size_t(n_strains));
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        sim_daycare_kernel<<<unsigned(B), 32, smem, stream>>>(a);
        return ELFI_B200_OK;
    });
}

int elfi_b200_daycare_summaries_f64(elfi_b200_ctx* ctx, const uint8_t* X, int64_t ld_b,
                                    int64_t ld_c, int64_t ld_i, int64_t ld_s, int64_t B,
                                    int64_t n_dcc, int64_t n_obs, int64_t n_strains, double* S,
                                    int64_t ldS, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || (X && S)), "daycare_summaries: NULL argument");
    ELFI_REQUIRE(B >= 0 && n_dcc >= 1 && n_obs >= 1 && n_strains >= 1 &&
                     n_strains <= ELFI_B200_DC_SUMM_STRAINS_MAX && ldS >= DC_NSUMM * n_dcc,
                 "daycare_summaries: bad shape (n_dcc, n_obs >= 1, 1 <= n_strains <= 64, "
                 "ldS >= 4 n_dcc; n_dcc=%lld n_obs=%lld n_strains=%lld ldS=%lld)",
                 (long long)n_dcc, (long long)n_obs, (long long)n_strains, (long long)ldS);
    if (B == 0) return ELFI_B200_OK;
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        const unsigned blocks = capped_grid(ctx, B * n_dcc, DC_SUMM_THREADS, 32);
        daycare_summaries_kernel<<<blocks, DC_SUMM_THREADS, 0, stream>>>(
            X, ld_b, ld_c, ld_i, ld_s, B, int(n_dcc), int(n_obs), int(n_strains), S, ldS);
        return ELFI_B200_OK;
    });
}

int elfi_b200_daycare_distance_f64(elfi_b200_ctx* ctx, const double* S, int64_t ldS, int64_t B,
                                   int64_t n_ss, int64_t n_dcc, const double* obs_max,
                                   const double* y, double* d, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || (S && obs_max && y && d)), "daycare_distance: NULL argument");
    ELFI_REQUIRE(B >= 0 && n_ss >= 1 && n_dcc >= 1 && n_ss * n_dcc <= DC_DIST_TERMS_MAX &&
                     ldS >= n_ss * n_dcc,
                 "daycare_distance: bad shape (n_ss * n_dcc <= %d, ldS >= n_ss * n_dcc; n_ss=%lld "
                 "n_dcc=%lld ldS=%lld)", DC_DIST_TERMS_MAX, (long long)n_ss, (long long)n_dcc,
                 (long long)ldS);
    if (B == 0) return ELFI_B200_OK;
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        const unsigned blocks = capped_grid(ctx, B, DC_DIST_THREADS, 32);
        daycare_distance_kernel<<<blocks, DC_DIST_THREADS, 0, stream>>>(
            S, ldS, B, int(n_ss), int(n_dcc), obs_max, y, d);
        return ELFI_B200_OK;
    });
}

}  // extern "C"
