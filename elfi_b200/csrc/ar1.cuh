// ar1.cuh -- the arithmetic of the AR(1) model of elfi/examples/ar1.py, shared by the device kernel
// (ar1.cu) and the host build of the tests (tests/harness/ar1_harness.cpp, g++ -ffp-contract=off):
// the recursion step and the Euclidean distance of the series to an observed one.
//
// Every operation is rounded on its own, as NumPy does it (ar1.py:30-38):
//   x_0 = 0,   x_t = phi * x_{t-1} + w_t,   t = 1 .. n_obs.
// The distance is SciPy's cdist 'euclidean' of the row to the observed row y (the order and the
// roundings that distance.cu states for its kernels):
//   acc = 0;  acc = acc + (x_t - y_t) * (x_t - y_t) for t ascending;  d = sqrt(acc).
// +, -, * and sqrt are correctly rounded on both sides, so a distance accumulated while the series
// is generated equals ops.dist_euclid of the written series bit for bit.
#pragma once

#include <math.h>

#include "hd.cuh"
#include "leafsum.cuh"

namespace elfi {

// x_t from x_{t-1} and the innovation w_t
ELFI_HD double ar1_step(double phi, double x_prev, double w) {
    return leaf_add(leaf_mul(phi, x_prev), w);
}

// the distance accumulator after the term of observation t: x_t against y_t
ELFI_HD double ar1_dist_term(double acc, double x, double y) {
    const double d = leaf_sub(x, y);
    return leaf_add(acc, leaf_mul(d, d));
}

// the distance from the accumulator of all terms (which starts at +0)
ELFI_HD double ar1_dist_finish(double acc) { return sqrt(acc); }

}  // namespace elfi
