// toad.cuh -- arithmetic of the toad movement model (elfi/examples/toad.py; Marchand et al. 2017):
// one symmetric alpha-stable step as SciPy 1.18's levy_stable.rvs computes it, the refuge day, and
// the per-count pieces of the displacement summaries as NumPy 2.3 computes them.  Every operation
// is rounded on its own (no FMA): leaf_add / leaf_sub / leaf_mul / gnk_div are __dadd_rn & co. on
// the device and plain operators on the host, where tests/harness/toad_harness.cpp builds this
// header with -ffp-contract=off and checks it against NumPy.
//
// Step: stable.cuh's levy_stable draw with beta = 0, loc = 0, scale gamma, in S1 (SciPy's default):
// the beta0func branch for alpha != 1, alpha1func at alpha == 1, where the S1 shift
// 2 beta gamma log(gamma) / pi is NaN at gamma = 0 (0 * -inf).
//
// Summaries of one lag (compute_summaries): the kept set is the non-NaN |displacements| >= thd,
// sorted, n of them.  np.nanquantile (method 'linear'): vi = (n - 1) p, lo = floor(vi), hi = lo + 1,
// t = vi - lo; vi >= n - 1 takes lo = hi = n - 1 and t = vi + 1 (NumPy keeps the index -1);
// gnk_lerp interpolates.  np.nanmedian of the (n_rows, B) array: below 600 rows the masked-array
// median, (a + b) / 2 of the middle pair with a = b for odd n; from 600 rows np.median of the kept
// set, the middle element itself for odd n.  Gaps log(max(diff, exp(-20))), NaN propagating
// through the maximum; finally nan_to_num: NaN -> inf, inf -> DBL_MAX, -inf -> -DBL_MAX.
#pragma once

#include <float.h>
#include <math.h>
#include <stdint.h>

#include "hd.cuh"
#include "../../include/elfi_b200.h"
#include "gnkstats.cuh"
#include "stable.cuh"

namespace elfi {

// displacements of one lag: n_toads * (n_days - lag)
constexpr int TOAD_DISP_MAX = ELFI_B200_TOAD_DISP_MAX;
constexpr int TOAD_NP_MAX = ELFI_B200_TOAD_NP_MAX;            // quantile levels
constexpr int TOAD_LAGS_MAX = ELFI_B200_TOAD_LAGS_MAX;           // lags of the fused summaries
constexpr int TOAD_MEDIAN_SMALL = 600;     // below: np.ma.median; from here: np.median
// n_days * n_toads: (cell << 1) | h < 2^32
constexpr int64_t TOAD_CELLS_MAX = ELFI_B200_TOAD_CELLS_MAX;
constexpr double TOAD_GAP_FLOOR = 0x1.1b48655f37267p-29;   // np.exp(-20)

ELFI_HD double toad_log(double x) { return log(x); }

// the reference raises for these (levy_stable's argcheck and scale >= 0); the device gives NaN rows
ELFI_HD bool toad_params_ok(double alpha, double gamma) {
    return stable_params_ok(alpha, 0.0, gamma);
}

ELFI_HD double toad_theta(double u) { return stable_theta(u); }
ELFI_HD double toad_expon(double u) { return stable_expon(u); }

// the per-toad factors of levy_stable.rvs(alpha, beta=0, scale=gamma) (S1)
ELFI_HD StableRow toad_stable_row(double alpha, double gamma) {
    return stable_row(alpha, 0.0, 0.0, gamma, false);
}

// levy_stable.rvs(alpha, beta=0, scale=gamma) (S1) of one (TH, W)
ELFI_HD double toad_stable_step(double alpha, double gamma, double TH, double W) {
    return stable_draw(toad_stable_row(alpha, gamma), TH, W);
}

// a refuge day uniform in [0, d) from a 64-bit word: the high word of w * d (bias below d / 2^64)
ELFI_HD int toad_refuge_day(uint64_t w, int d) {
#if defined(__CUDA_ARCH__)
    return int(__umul64hi(w, uint64_t(d)));
#else
    return int((unsigned __int128)w * uint64_t(d) >> 64);
#endif
}

// np.nanquantile's picks over a sorted kept set of n >= 1 values
struct ToadPick {
    int lo, hi;
    double t;
};
ELFI_HD ToadPick toad_quantile_pick(int n, double p) {
    const double vi = leaf_mul(double(n - 1), p);
    ToadPick r;
    if (vi >= double(n - 1)) {
        r.lo = r.hi = n - 1;
        r.t = leaf_sub(vi, -1.0);
    } else {
        const double f = floor(vi);
        r.lo = int(f);
        r.hi = r.lo + 1;
        r.t = leaf_sub(vi, f);
    }
    return r;
}

// middle positions of the median of n >= 1 sorted values: (lo, hi); odd n has lo == hi
ELFI_HD void toad_median_picks(int n, int& lo, int& hi) {
    hi = n / 2;
    lo = (n & 1) ? hi : hi - 1;
}

// the median from the middle values a = sorted[lo], b = sorted[hi] (see toad_median_picks)
ELFI_HD double toad_median(double a, double b, int n, int n_rows) {
    if ((n & 1) && n_rows >= TOAD_MEDIAN_SMALL) return a;
    return gnk_div(leaf_add(a, b), 2.0);
}

ELFI_HD double toad_nan_to_num(double x) {
    if (x != x) return INFINITY;
    if (x == INFINITY) return DBL_MAX;
    if (x == -INFINITY) return -DBL_MAX;
    return x;
}

// np.log(np.maximum(hi - lo, np.exp(-20))), before nan_to_num
ELFI_HD double toad_log_gap(double lo, double hi) {
    const double d = leaf_sub(hi, lo);
    return toad_log((d != d) ? d : (d >= TOAD_GAP_FLOOR ? d : TOAD_GAP_FLOOR));
}

}  // namespace elfi
