// rowquantiles.cuh -- np.quantile (method 'linear') of a row that one warp holds in registers, shared
// by the M/G/1 kernels (mg1.cu: the fused quantiles and row_quantiles) and the stochastic
// volatility model's fused kurtosis and skewness (svm.cu).  The row's n <= MG1_NOBS_MAX keys
// (bitonic.cuh's order-preserving u64, padding ~0) are sorted by bitonic_in_registers; lane k then
// picks and interpolates level k (mg1.cuh's toad_quantile_pick and gnk_lerp).  A row containing NaN
// has every quantile NaN (NaN sorts last, NumPy checks the last element).  kpl_for also sizes the
// register rows of the g-and-k summaries (gnkstats.cu).
#pragma once

#include <string.h>

#include "bitonic.cuh"
#include "mg1.cuh"

namespace elfi {

struct QuantileLevels {
    double q[MG1_NQ_MAX];
};

// keys per lane of a row of n values that a warp holds in registers: the least power of two
// kpl >= min_kpl with 32 * kpl >= n
static inline int kpl_for(int n, int min_kpl) {
    int kpl = min_kpl;
    while (32 * kpl < n) kpl <<= 1;
    return kpl;
}

// The per-warp strips of the one-thread-per-row simulators (mg1.cu, svm.cu): thread r of a warp
// writes its row of n values to strip[r * npad + j], npad = n | 1 (an odd stride: no bank
// conflicts), and a block of 32 * warps threads has as many warps (1 .. warps_max) as fit in
// `budget` bytes of shared memory.
struct WarpStrips {
    int npad, warps;
    size_t smem;        // dynamic shared memory of a block
    unsigned blocks;    // blocks that cover B rows
};

static inline WarpStrips warp_strips(int64_t B, int n, size_t budget, int warps_max) {
    WarpStrips s;
    s.npad = n | 1;
    const size_t warp_bytes = size_t(32) * s.npad * sizeof(double);
    const int warps = int(budget / warp_bytes);
    s.warps = warps < 1 ? 1 : (warps > warps_max ? warps_max : warps);
    s.smem = s.warps * warp_bytes;
    s.blocks = unsigned((B + 32 * s.warps - 1) / (32 * s.warps));
    return s;
}

// the levels as the kernels take them; false if one lies outside [0, 1] (or is NaN)
static inline bool quantile_levels(const double* q_host, int64_t nq, QuantileLevels* Q) {
    memset(Q, 0, sizeof(*Q));
    for (int k = 0; k < nq; ++k) {
        if (!(q_host[k] >= 0.0 && q_host[k] <= 1.0)) return false;
        Q->q[k] = q_host[k];
    }
    return true;
}

// sort a register-resident row of n keys (padding ~0) and return the quantile of the lane's pick
// pk (every lane of the warp calls it)
template <int KPL>
__device__ __forceinline__ double quantile_of_keys(uint64_t (&key)[KPL], int lane, int n,
                                                   const ToadPick& pk) {
    bitonic_in_registers<KPL>(key, lane);
    const bool has_nan = pick_reg(key, n - 1) == ~uint64_t(0);
    const double a = u64_to_key(pick_reg_lane(key, pk.lo));
    const double b = u64_to_key(pick_reg_lane(key, pk.hi));
    return has_nan ? NAN : gnk_lerp(a, b, pk.t);
}

// sort a register-resident row of n keys (padding ~0) and write quantile `lane` to S_row[lane]
// for lane < nq (pk: the lane's pick)
template <int KPL>
__device__ __forceinline__ void quantiles_of_keys(uint64_t (&key)[KPL], int lane, int n, int nq,
                                                  const ToadPick& pk, bool live, double* S_row) {
    const double v = quantile_of_keys<KPL>(key, lane, n, pk);
    if (live && lane < nq) S_row[lane] = v;
}

// the pick of level `lane` (level 0 for lanes >= nq, whose value nobody writes)
__device__ __forceinline__ ToadPick lane_pick(int n, int nq, const QuantileLevels& Q, int lane) {
    double q = Q.q[0];
#pragma unroll
    for (int k = 1; k < MG1_NQ_MAX; ++k)
        if (k == lane && k < nq) q = Q.q[k];
    return toad_quantile_pick(n, q);
}

}  // namespace elfi
