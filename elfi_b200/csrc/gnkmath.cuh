// gnkmath.cuh -- quantile function of the g-and-k distribution (elfi/examples/gnk.py:11-68):
//   y = A + B * (1 + c * (1 - exp(-g z)) / (1 + exp(-g z))) * (1 + z^2)^k * z,   z ~ N(0, 1)
// evaluated in the reference's operation order.  Compiles for the host as well
// (tests/harness/gnk_harness.cpp checks it against the NumPy expression on a CPU).
#pragma once

#include <math.h>

#include "hd.cuh"

namespace elfi {

ELFI_HD double gnk_quantile(double A, double B, double g, double k, double c, double z) {
    const double e = exp(-g * z);
    const double skew = 1.0 + c * ((1.0 - e) / (1.0 + e));
    const double kurt = pow(1.0 + z * z, k);
    return A + ((B * skew) * kurt) * z;
}

}  // namespace elfi
