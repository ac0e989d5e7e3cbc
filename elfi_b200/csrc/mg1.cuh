// mg1.cuh -- the arithmetic of the M/G/1 queue of elfi/examples/mg1.py, shared by the device
// kernels (mg1.cu) and the host build of the tests (tests/harness/mg1_harness.cpp, g++
// -ffp-contract=off): the inter-arrival and service times from uniforms, the queue recurrence and
// the quantile picks.
//
// Every operation is rounded on its own, in the reference's order (mg1.py:37-54):
//   W_i = (1 / t3) * (-log u)               RandomState.exponential(1/t3): scale * (-log(1 - u0))
//   U_i = t1 + (t2 - t1) * u'               RandomState.uniform(t1, t2): low + range * u0
//   sum_w += W_i;  y_i = U_i + max(0, sum_w - sum_x);  sum_x += y_i
// with u, u' uniform on (0, 1] from the device streams.  The max is np.maximum(0, d): d itself
// unless d < 0, so NaN propagates and -0.0 passes through (CUDA's fmax(0, NaN) returns 0, the
// wrong operation here).  Rows where NumPy raises -- 1/t3 with its sign bit set (NumPy refuses a
// scale < 0 by its sign bit, so t3 = -0.0 and t3 = -inf are refused too) or t2 - t1 not finite
// (OverflowError) -- give NaN data; every other edge follows NumPy's arithmetic (t3 = 0 gives
// infinite gaps, t3 = NaN NaN ones).
//
// Quantiles (mg1.py:62-65, np.quantile(x, q, axis=1), method 'linear') of a sorted row of n
// values: toad_quantile_pick's lo, hi and t, then gnk_lerp; a row containing NaN has every quantile
// NaN (NaN sorts last, NumPy checks the last element).
#pragma once

#include <math.h>
#include <stdint.h>

#include "hd.cuh"
#include "../../include/elfi_b200.h"
#include "gnkstats.cuh"
#include "toad.cuh"

namespace elfi {

constexpr int MG1_NOBS_MIN = ELFI_B200_MG1_NOBS_MIN;
// one warp sorts a row in registers (32 lanes x 16 keys)
constexpr int MG1_NOBS_MAX = ELFI_B200_MG1_NOBS_MAX;
constexpr int MG1_NQ_MAX = ELFI_B200_MG1_NQ_MAX;      // one quantile per lane

// false where the reference raises: the row is NaN
ELFI_HD bool mg1_params_ok(double inv_t3, double range) {
    return !(signbit(inv_t3) && inv_t3 == inv_t3) && isfinite(range);
}

// the inter-arrival time from u in (0, 1]
ELFI_HD double mg1_gap(double inv_t3, double u) { return leaf_mul(inv_t3, -log(u)); }

// the service time from u in (0, 1]
ELFI_HD double mg1_service(double t1, double range, double u) {
    return leaf_add(t1, leaf_mul(range, u));
}

// np.maximum(0, d)
ELFI_HD double mg1_max0(double d) { return d < 0.0 ? 0.0 : d; }

// one customer: updates the running arrival and departure sums, returns the inter-departure time
ELFI_HD double mg1_step(double& sum_w, double& sum_x, double W, double U) {
    sum_w = leaf_add(sum_w, W);
    const double y = leaf_add(U, mg1_max0(leaf_sub(sum_w, sum_x)));
    sum_x = leaf_add(sum_x, y);
    return y;
}

// quantile q of a sorted row of n values: sorted(i) returns the value at sorted position i
template <class Sorted>
ELFI_HD double mg1_quantile(int n, double q, const Sorted& sorted) {
    const ToadPick pk = toad_quantile_pick(n, q);
    if (sorted(n - 1) != sorted(n - 1)) return NAN;
    return gnk_lerp(sorted(pk.lo), sorted(pk.hi), pk.t);
}

}  // namespace elfi
