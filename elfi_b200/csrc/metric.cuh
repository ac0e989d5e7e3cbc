// metric.cuh -- the per-term arithmetic and the finish of the unweighted cdist metrics, shared by
// the distance kernels (distance.cu) and the all-combination distances (sumsel.cu).
//
// SciPy 1.18 accumulates 'euclidean', 'sqeuclidean', 'cityblock', 'chebyshev' and 'minkowski' left
// to right in fp64 (probed: bit-identical to a sequential loop at 2000 x 128).  Every multiply and
// add is rounded on its own (__dmul_rn / __dadd_rn), so nvcc cannot contract them into FMA.
#pragma once

#include "common.cuh"

namespace elfi {

// acc after one more term d = x_j - obs_j.  'chebyshev' keeps acc when d is NaN, like SciPy's
// std::max(acc, |d|).
template <int METRIC>
__device__ __forceinline__ double metric_term(double acc, double d, double pexp) {
    if (METRIC == ELFI_B200_METRIC_EUCLIDEAN || METRIC == ELFI_B200_METRIC_SQEUCLIDEAN)
        return __dadd_rn(acc, __dmul_rn(d, d));
    if (METRIC == ELFI_B200_METRIC_CITYBLOCK) return __dadd_rn(acc, fabs(d));
    if (METRIC == ELFI_B200_METRIC_CHEBYSHEV) return fabs(d) > acc ? fabs(d) : acc;
    return __dadd_rn(acc, pow(fabs(d), pexp));                       // Minkowski
}

// The distance from the accumulator of all terms (which starts at +0).
template <int METRIC>
__device__ __forceinline__ double metric_value(double acc, double pexp) {
    if (METRIC == ELFI_B200_METRIC_EUCLIDEAN) return sqrt(acc);
    return METRIC == ELFI_B200_METRIC_MINKOWSKI ? pow(acc, 1.0 / pexp) : acc;
}

}  // namespace elfi
