// toad.cuh -- arithmetic of the toad movement model (elfi/examples/toad.py; Marchand et al. 2017):
// one symmetric alpha-stable step as SciPy 1.18's levy_stable.rvs computes it, the refuge day, and
// the per-count pieces of the displacement summaries as NumPy 2.3 computes them.  Every operation
// is rounded on its own (no FMA): leaf_add / leaf_sub / leaf_mul / gnk_div are __dadd_rn & co. on
// the device and plain operators on the host, where tests/harness/toad_harness.cpp builds this
// header with -ffp-contract=off and checks it against NumPy.
//
// Step (scipy/stats/_levy_stable: _rvs_Z1 with beta = 0, then vals * scale + loc and the S1 shift
// of levy_stable_gen.rvs), from TH uniform on (-pi/2, pi/2) and W standard exponential:
//   alpha != 1  (beta0func)   W / (cos TH / tan(aTH) + sin TH) * ((cos aTH + sin aTH tan TH) / W) ** (1 / alpha)
//   alpha == 1  (alpha1func)  2 / pi * ((pi / 2 + bTH) tan TH - beta log((pi / 2 W cos TH) / (pi / 2 + bTH)))
//   with aTH = alpha TH, bTH = beta TH = +-0; then X = vals * gamma + 0, and at alpha == 1
//   X + 2 beta gamma log(gamma) / pi, which is NaN at gamma = 0 (0 * -inf).
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

#include "gnkstats.cuh"

namespace elfi {

constexpr int TOAD_DISP_MAX = 4096;        // displacements of one lag: n_toads * (n_days - lag)
constexpr int TOAD_NP_MAX = 32;            // quantile levels
constexpr int TOAD_LAGS_MAX = 8;           // lags of the fused summaries
constexpr int TOAD_MEDIAN_SMALL = 600;     // below: np.ma.median; from here: np.median
constexpr int64_t TOAD_CELLS_MAX = int64_t(1) << 31;   // n_days * n_toads: (cell << 1) | h < 2^32
constexpr double TOAD_GAP_FLOOR = 0x1.1b48655f37267p-29;   // np.exp(-20)
constexpr double TOAD_PI = 3.141592653589793;           // np.pi
constexpr double TOAD_PI_2 = 1.5707963267948966;        // np.pi / 2

ELFI_HD double toad_sin(double x) { return sin(x); }
ELFI_HD double toad_cos(double x) { return cos(x); }
ELFI_HD double toad_tan(double x) { return tan(x); }
ELFI_HD double toad_log(double x) { return log(x); }
ELFI_HD double toad_pow(double x, double y) { return pow(x, y); }

// the reference raises for these (levy_stable's argcheck and scale >= 0); the device gives NaN rows
ELFI_HD bool toad_params_ok(double alpha, double gamma) {
    return alpha > 0.0 && alpha <= 2.0 && gamma >= 0.0;
}

// TH = uniform.rvs(loc=-pi/2, scale=pi) from u in [0, 1): u * pi + (-pi / 2)
ELFI_HD double toad_theta(double u) { return leaf_add(leaf_mul(u, TOAD_PI), -TOAD_PI_2); }
// W = expon.rvs() from u in (0, 1]: -log(u) * 1 + 0
ELFI_HD double toad_expon(double u) { return leaf_add(leaf_mul(-toad_log(u), 1.0), 0.0); }

// levy_stable.rvs(alpha, beta=0, scale=gamma) (S1) of one (TH, W)
ELFI_HD double toad_stable_step(double alpha, double gamma, double TH, double W) {
    const double aTH = leaf_mul(alpha, TH);
    const double cosTH = toad_cos(TH), tanTH = toad_tan(TH);
    double val;
    if (alpha == 1.0) {
        const double bTH = leaf_mul(0.0, TH);
        const double h = leaf_add(TOAD_PI_2, bTH);
        const double lg = toad_log(gnk_div(leaf_mul(leaf_mul(TOAD_PI_2, W), cosTH), h));
        val = leaf_mul(2.0 / TOAD_PI, leaf_sub(leaf_mul(h, tanTH), leaf_mul(0.0, lg)));
    } else {
        const double den = leaf_add(gnk_div(cosTH, toad_tan(aTH)), toad_sin(TH));
        const double num = leaf_add(toad_cos(aTH), leaf_mul(toad_sin(aTH), tanTH));
        val = leaf_mul(gnk_div(W, den), toad_pow(gnk_div(num, W), gnk_div(1.0, alpha)));
    }
    double x = leaf_add(leaf_mul(val, gamma), 0.0);
    if (alpha == 1.0)
        x = leaf_add(x, gnk_div(leaf_mul(leaf_mul(0.0, gamma), toad_log(gamma)), TOAD_PI));
    return x;
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
