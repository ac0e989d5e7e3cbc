// svm.cuh -- the arithmetic of the alpha-stable stochastic volatility model of
// elfi/examples/stochastic_volatility_model.py, shared by the device kernel (svm.cu) and the host
// build of the tests (tests/harness/svm_harness.cpp, g++ -ffp-contract=off).  Every operation is
// rounded on its own, in the reference's order:
//   log-volatility  x_0 = z_0 * s + mu,  s = sigma / sqrt(1 - min(phi ** 2, 0.99999))
//                   x_t = z_t * sigma + (mu + phi * (x_{t-1} - mu))    (norm.rvs: z * scale + loc)
//   shock           v_t = levy_stable(alpha, beta, loc=eta, scale=kappa) in S0 (stable.cuh)
//   data            y_t = exp(0.5 * x_t) * v_t
// Rows where the reference raises -- levy_stable's argcheck (0 < alpha <= 2, -1 <= beta <= 1),
// kappa < 0, or a norm.rvs scale < 0 (sigma < 0, or a stationary scale that is NaN, e.g. phi = NaN)
// -- give NaN data; every other edge follows the arithmetic.
//
// Summaries of a sorted row of n values (np.quantile, method 'linear'; the levels 0.05, 0.25, 0.5,
// 0.75, 0.95 are picked exactly as the reference's two separate np.quantile calls pick them):
//   kurt = (q95 - q05) / (q75 - q25),   skew = ((q95 - q50) - (q50 - q05)) / (q95 - q05).
#pragma once

#include <math.h>

#include "hd.cuh"
#include "gnkstats.cuh"
#include "stable.cuh"
#include "toad.cuh"

namespace elfi {

constexpr int SVM_NPARAMS = 7;      // alpha, beta, kappa, eta, mu, phi, sigma
constexpr int SVM_NSUMM = 2;        // kurt, skew
constexpr int SVM_NQ = 5;           // the quantile levels of the two summaries
constexpr double SVM_PHI2_MAX = 0.99999;

// the levels, in the order svm_kurt / svm_skew take them
ELFI_HD double svm_level(int k) {
    return k == 0 ? 0.05 : k == 1 ? 0.25 : k == 2 ? 0.5 : k == 3 ? 0.75 : 0.95;
}

// sigma / sqrt(1 - min(phi ** 2, 0.99999)), the scale of x_0 (np.minimum propagates NaN)
ELFI_HD double svm_stationary_scale(double phi, double sigma) {
    const double p2 = leaf_mul(phi, phi);
    const double m = (p2 != p2) ? p2 : (p2 < SVM_PHI2_MAX ? p2 : SVM_PHI2_MAX);
    return gnk_div(sigma, sqrt(leaf_sub(1.0, m)));
}

// false where the reference raises: the row is NaN
ELFI_HD bool svm_params_ok(double alpha, double beta, double kappa, double sigma, double scale0) {
    return stable_params_ok(alpha, beta, kappa) && sigma >= 0.0 && scale0 >= 0.0;
}

// x_0 from its normal
ELFI_HD double svm_x0(double z, double mu, double scale0) {
    return leaf_add(leaf_mul(z, scale0), mu);
}

// x_t from x_{t-1} and its normal
ELFI_HD double svm_ar1(double z, double x_prev, double mu, double phi, double sigma) {
    return leaf_add(leaf_mul(z, sigma), leaf_add(mu, leaf_mul(phi, leaf_sub(x_prev, mu))));
}

// y_t = exp(0.5 x_t) v_t
ELFI_HD double svm_y(double x, double v) { return leaf_mul(exp(leaf_mul(0.5, x)), v); }

ELFI_HD double svm_kurt(double q05, double q25, double q75, double q95) {
    return gnk_div(leaf_sub(q95, q05), leaf_sub(q75, q25));
}

ELFI_HD double svm_skew(double q05, double q50, double q95) {
    return gnk_div(leaf_sub(leaf_sub(q95, q50), leaf_sub(q50, q05)), leaf_sub(q95, q05));
}

}  // namespace elfi
