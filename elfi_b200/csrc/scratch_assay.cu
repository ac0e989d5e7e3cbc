// scratch_assay.cu -- the scratch assay model of elfi/examples/scratch_assay.py in throughput mode:
// the lattice simulator with its mismatch summaries fused, and the summaries of given data.  The
// law and the stream layout are in scratch_assay.cuh.
//
// Layout: one warp per row, its state in shared memory: the bit-packed lattice (W = ceil(N / 32)
// words), the previous frame's words and the uint16 snapshot list (N entries); about 2.2 KB per
// row at 27 x 36.  Each iteration:
//   * the snapshot: each lane takes one word per round, a warp scan of the popcounts gives its
//     offset, and it writes its set bits' sites in order, so the list is row-major;
//   * each phase tests 32 slots at a time, one Philox block per lane.  Motility applies the kept
//     slots of a ballot in slot order on lane 0 (each depends on the lattice the previous one
//     left); proliferation only sets bits, so every kept lane sets its target with a shared-memory
//     atomicOr;  a phase whose probability is not > 0 keeps no slot and is skipped;
//   * at each observation the mismatch popcount(prev ^ cur) is reduced over the warp and the
//     current words become prev.  The frame goes to X only when X is asked for.
// A full lattice never changes again, so the row then skips to its remaining observations.
#include "common.cuh"
#include "scratch_assay.cuh"

namespace elfi {

constexpr int SA_WARPS = 4;
constexpr int SA_SUMM_THREADS = 256;
constexpr unsigned SA_FULL_MASK = 0xffffffffu;

struct SaSim {
    const double* P;
    int64_t ldP;
    int64_t B;
    const uint8_t* init;
    int nrows, ncols, num_obs, interval;
    uint64_t seed, offset;
    double* S;
    int64_t ldS;
    uint8_t* X;
};

// 32-bit words of shared memory one row needs: lattice, previous frame, list
__host__ __device__ inline int sa_row_words(int nsites) { return 2 * sa_words(nsites) + (nsites + 1) / 2; }

__device__ __forceinline__ int sa_warp_sum(int v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(SA_FULL_MASK, v, o);
    return v;
}

__device__ __forceinline__ void sa_write_frame(const SaSim& a, int64_t i, int k, int N, int lane,
                                               const uint32_t* lat) {
    uint8_t* x = a.X + size_t(i) * N * (a.num_obs + 1) + k;
    for (int s = lane; s < N; s += 32) x[size_t(s) * (a.num_obs + 1)] = uint8_t(sa_get(lat, s));
}

__global__ void __launch_bounds__(32 * SA_WARPS) sim_scratch_assay_kernel(SaSim a) {
    extern __shared__ uint32_t sa_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t i = int64_t(blockIdx.x) * SA_WARPS + warp;
    if (i >= a.B) return;                                   // warp-uniform
    const int N = a.nrows * a.ncols, W = sa_words(N);
    uint32_t* lat = sa_smem + size_t(warp) * sa_row_words(N);
    uint32_t* prev = lat + W;
    uint16_t* list = reinterpret_cast<uint16_t*>(prev + W);
    const double pm = a.P[i * a.ldP], pp = a.P[i * a.ldP + 1];
    const Philox ph(a.seed);
    const uint64_t row = a.offset + uint64_t(i);

    for (int w = lane; w < W; w += 32) {
        uint32_t bits = 0;
        for (int b = 0; b < 32 && w * 32 + b < N; ++b) bits |= uint32_t(a.init[w * 32 + b] != 0) << b;
        lat[w] = prev[w] = bits;
    }
    __syncwarp();
    if (a.X) sa_write_frame(a, i, 0, N, lane, lat);

    bool full = false;
    const int iters = a.num_obs * a.interval;
    for (int t = 0; t < iters; ++t) {
        if (full) {
            t = (t / a.interval + 1) * a.interval - 1;      // nothing changes until the next frame
        } else {
            int n = 0;
            for (int base = 0; base < W; base += 32) {
                const int w = base + lane;
                uint32_t bits = w < W ? lat[w] : 0u;
                const int c = __popc(bits);
                int incl = c;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const int v = __shfl_up_sync(SA_FULL_MASK, incl, o);
                    if (lane >= o) incl += v;
                }
                int pos = n + incl - c;
                for (; bits; bits &= bits - 1) list[pos++] = uint16_t(w * 32 + __ffs(bits) - 1);
                n += __shfl_sync(SA_FULL_MASK, incl, 31);
            }
            __syncwarp();
            if (n == N) {
                full = true;
            } else {
                if (pm > 0) {
                    for (int base = 0; base < n; base += 32) {
                        const int s = base + lane;
                        SaSlot sl = {false, 0, 0};
                        if (s < n) sl = sa_slot(ph, row, t, 0, s, n, pm);
                        for (uint32_t kept = __ballot_sync(SA_FULL_MASK, sl.kept); kept;
                             kept &= kept - 1) {
                            const int l = __ffs(kept) - 1;
                            const int idx = __shfl_sync(SA_FULL_MASK, sl.index, l);
                            const int dir = __shfl_sync(SA_FULL_MASK, sl.dir, l);
                            if (lane == 0) {
                                const int from = list[idx];
                                const int to = sa_target(from, dir, a.nrows, a.ncols);
                                if (!sa_get(lat, to)) {
                                    lat[from >> 5] &= ~(1u << (from & 31));
                                    lat[to >> 5] |= 1u << (to & 31);
                                    list[idx] = uint16_t(to);
                                }
                            }
                        }
                    }
                    __syncwarp();
                }
                if (pp > 0) {
                    for (int s = lane; s < n; s += 32) {
                        const SaSlot sl = sa_slot(ph, row, t, 1, s, n, pp);
                        if (sl.kept) {
                            const int to = sa_target(list[sl.index], sl.dir, a.nrows, a.ncols);
                            atomicOr(&lat[to >> 5], 1u << (to & 31));
                        }
                    }
                    __syncwarp();
                }
            }
        }
        if ((t + 1) % a.interval == 0) {
            const int k = (t + 1) / a.interval;
            int m = 0;
            for (int w = lane; w < W; w += 32) {
                const uint32_t cur = lat[w];
                m += __popc(cur ^ prev[w]);
                prev[w] = cur;
            }
            m = sa_warp_sum(m);
            if (a.S && lane == 0) a.S[i * a.ldS + (k - 1)] = double(m);
            if (a.X) sa_write_frame(a, i, k, N, lane, lat);
            __syncwarp();
        }
    }
    if (a.S) {
        int count = 0;
        for (int w = lane; w < W; w += 32) count += __popc(prev[w]);
        count = sa_warp_sum(count);
        if (lane == 0) a.S[i * a.ldS + a.num_obs] = double(count);
    }
}

// S[b, k] = the mismatch between frames k and k + 1 (k < F - 1), S[b, F - 1] = the cells of the
// last frame; one thread per (row, column), nonzero meaning a cell
__global__ void __launch_bounds__(SA_SUMM_THREADS)
scratch_assay_summaries_kernel(const uint8_t* __restrict__ X, int64_t ld_b, int64_t ld_r,
                               int64_t ld_c, int64_t ld_k, int64_t B, int nrows, int ncols, int F,
                               double* __restrict__ S, int64_t ldS) {
    const int64_t total = B * F, stride = int64_t(gridDim.x) * blockDim.x;
    for (int64_t e = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; e < total; e += stride) {
        const int64_t b = e / F;
        const int k = int(e - b * F);
        const uint8_t* x = X + b * ld_b + k * ld_k;
        int64_t sum = 0;
        for (int r = 0; r < nrows; ++r)
            for (int c = 0; c < ncols; ++c) {
                const uint8_t* p = x + r * ld_r + c * ld_c;
                sum += k + 1 < F ? int((p[0] != 0) != (p[ld_k] != 0)) : int(p[0] != 0);
            }
        S[b * ldS + k] = double(sum);
    }
}

}  // namespace elfi

extern "C" {

int elfi_b200_sim_scratch_assay_f64(elfi_b200_ctx* ctx, const double* P, int64_t ldP, int64_t B,
                                    const uint8_t* init, int64_t nrows, int64_t ncols,
                                    int64_t num_iter, int64_t obs_interval, uint64_t seed,
                                    uint64_t offset, double* S, int64_t ldS, uint8_t* X,
                                    void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || (P && init)), "sim_scratch_assay: NULL argument");
    ELFI_REQUIRE(B >= 0 && B <= ELFI_B200_SA_BATCH_MAX && ldP >= SA_NPARAMS && nrows >= 1 &&
                     ncols >= 1 && nrows <= SA_SITES_MAX && ncols <= SA_SITES_MAX &&
                     nrows * ncols <= SA_SITES_MAX && num_iter >= 0 &&
                     num_iter <= ELFI_B200_SA_ITER_MAX &&
                     obs_interval >= 1 && (S == nullptr || ldS >= num_iter / obs_interval + 1),
                 "sim_scratch_assay: bad shape (1 <= nrows * ncols <= %d, 0 <= num_iter < 2^31, "
                 "obs_interval >= 1, ldS >= num_iter / obs_interval + 1, B < 2^31; B=%lld "
                 "nrows=%lld ncols=%lld num_iter=%lld obs_interval=%lld ldS=%lld)", SA_SITES_MAX,
                 (long long)B, (long long)nrows, (long long)ncols, (long long)num_iter,
                 (long long)obs_interval, (long long)ldS);
    if (B == 0 || (S == nullptr && X == nullptr)) return ELFI_B200_OK;
    SaSim a;
    a.P = P;
    a.ldP = ldP;
    a.B = B;
    a.init = init;
    a.nrows = int(nrows);
    a.ncols = int(ncols);
    a.num_obs = int(num_iter / obs_interval);
    a.interval = int(obs_interval);
    a.seed = seed;
    a.offset = offset;
    a.S = S;
    a.ldS = ldS;
    a.X = X;
    const size_t smem = size_t(SA_WARPS) * sa_row_words(int(nrows * ncols)) * sizeof(uint32_t);
    const unsigned blocks = unsigned((B + SA_WARPS - 1) / SA_WARPS);
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        sim_scratch_assay_kernel<<<blocks, 32 * SA_WARPS, smem, stream>>>(a);
        return ELFI_B200_OK;
    });
}

int elfi_b200_scratch_assay_summaries_f64(elfi_b200_ctx* ctx, const uint8_t* X, int64_t ld_b,
                                          int64_t ld_r, int64_t ld_c, int64_t ld_k, int64_t B,
                                          int64_t nrows, int64_t ncols, int64_t n_frames,
                                          double* S, int64_t ldS, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || (X && S)), "scratch_assay_summaries: NULL argument");
    ELFI_REQUIRE(B >= 0 && nrows >= 1 && ncols >= 1 && n_frames >= 1 &&
                     n_frames <= 0x7fffffff && ldS >= n_frames,
                 "scratch_assay_summaries: bad shape (nrows, ncols, n_frames >= 1, ldS >= "
                 "n_frames; nrows=%lld ncols=%lld n_frames=%lld ldS=%lld)", (long long)nrows,
                 (long long)ncols, (long long)n_frames, (long long)ldS);
    if (B == 0) return ELFI_B200_OK;
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        const unsigned blocks = capped_grid(ctx, B * n_frames, SA_SUMM_THREADS, 32);
        scratch_assay_summaries_kernel<<<blocks, SA_SUMM_THREADS, 0, stream>>>(
            X, ld_b, ld_r, ld_c, ld_k, B, int(nrows), int(ncols), int(n_frames), S, ldS);
        return ELFI_B200_OK;
    });
}

}  // extern "C"
