// stable.cuh -- one alpha-stable draw as SciPy 1.18's levy_stable.rvs computes it, for any (alpha,
// beta), in the S1 or the S0 parameterization: scipy/stats/_levy_stable's _rvs_Z1, then rv_generic's
// vals * scale + loc, then levy_stable_gen.rvs's location shifts.  Shared by the toad walk (toad.cuh,
// beta = 0, S1) and the stochastic volatility model (svm.cuh, S0).  Every operation is rounded on its
// own (no FMA): leaf_add / leaf_sub / leaf_mul / gnk_div are __dadd_rn & co. on the device and plain
// operators on the host, where tests/harness/svm_harness.cpp builds this header with
// -ffp-contract=off and checks it against a NumPy restatement of SciPy.
//
// From TH uniform on [-pi/2, pi/2) and W standard exponential, with aTH = alpha TH, bTH = beta TH,
// the branch chosen per element as SciPy's apply_where does (alpha == 1, else beta == 0 -- -0.0
// included -- else otherwise):
//   alpha == 1  2 / pi * ((pi / 2 + bTH) tan TH - beta log((pi / 2 W cos TH) / (pi / 2 + bTH)))
//   beta == 0   W / (cos TH / tan aTH + sin TH) * ((cos aTH + sin aTH tan TH) / W) ** (1 / alpha)
//   otherwise   val0 = beta tan(pi alpha / 2), th0 = arctan(val0) / alpha,
//               W / (cos TH / tan(alpha (th0 + TH)) + sin TH)
//                 * ((cos aTH + sin aTH tan TH - val0 (sin aTH - cos aTH tan TH)) / W) ** (1 / alpha)
// then X = Z1 * scale + loc; at alpha == 1 the S1 shift X + 2 beta scale log(scale) / pi; in S0,
// X - beta 2 scale log(scale) / pi at alpha == 1 (the same value: (X + a) - a, kept as two
// roundings), otherwise X - scale beta tan(pi alpha / 2).  NumPy evaluates these left to right and
// broadcasts the per-parameter factors, so hoisting them into StableRow gives the same bits.
#pragma once

#include <math.h>

#include "hd.cuh"
#include "gnkstats.cuh"

namespace elfi {

constexpr double STABLE_PI = 3.141592653589793;      // np.pi
constexpr double STABLE_PI_2 = 1.5707963267948966;   // np.pi / 2

ELFI_HD double stable_sin(double x) { return sin(x); }
ELFI_HD double stable_cos(double x) { return cos(x); }
ELFI_HD double stable_tan(double x) { return tan(x); }
ELFI_HD double stable_atan(double x) { return atan(x); }
ELFI_HD double stable_log(double x) { return log(x); }
ELFI_HD double stable_pow(double x, double y) { return pow(x, y); }

// levy_stable's argcheck (0 < alpha <= 2, -1 <= beta <= 1) and rv_generic's scale >= 0; NaN fails
ELFI_HD bool stable_params_ok(double alpha, double beta, double scale) {
    return alpha > 0.0 && alpha <= 2.0 && beta >= -1.0 && beta <= 1.0 && scale >= 0.0;
}

enum StableBranch { STABLE_ALPHA1 = 0, STABLE_BETA0 = 1, STABLE_OTHERWISE = 2 };

// the per-parameter factors of one draw, computed once per row
struct StableRow {
    double alpha, beta, loc, scale;
    double inv_alpha;    // 1.0 / alpha                              (alpha != 1)
    double val0, th0;    // beta tan(pi alpha / 2), arctan(val0) / alpha   (otherwise)
    double shift1;       // 2 beta scale log(scale) / pi             (alpha == 1)
    double shift0;       // the S0 shift subtracted last             (s0)
    int branch;
    bool s0;
};

ELFI_HD StableRow stable_row(double alpha, double beta, double loc, double scale, bool s0) {
    StableRow r;
    r.alpha = alpha;
    r.beta = beta;
    r.loc = loc;
    r.scale = scale;
    r.s0 = s0;
    r.branch = alpha == 1.0 ? STABLE_ALPHA1 : (beta == 0.0 ? STABLE_BETA0 : STABLE_OTHERWISE);
    r.inv_alpha = gnk_div(1.0, alpha);
    r.val0 = r.th0 = r.shift1 = r.shift0 = 0.0;
    const double tan_a = (r.branch == STABLE_OTHERWISE || (s0 && r.branch != STABLE_ALPHA1))
                             ? stable_tan(gnk_div(leaf_mul(STABLE_PI, alpha), 2.0)) : 0.0;
    if (r.branch == STABLE_OTHERWISE) {
        r.val0 = leaf_mul(beta, tan_a);
        r.th0 = gnk_div(stable_atan(r.val0), alpha);
    }
    if (r.branch == STABLE_ALPHA1) {
        r.shift1 = gnk_div(leaf_mul(leaf_mul(leaf_mul(2.0, beta), scale), stable_log(scale)),
                           STABLE_PI);
        r.shift0 = r.shift1;   // beta * 2 * scale * log(scale) / pi: 2 beta == beta 2 exactly
    } else if (s0) {
        r.shift0 = leaf_mul(leaf_mul(scale, beta), tan_a);
    }
    return r;
}

// TH = uniform.rvs(loc=-pi/2, scale=pi) from u in [0, 1): u * pi + (-pi / 2)
ELFI_HD double stable_theta(double u) { return leaf_add(leaf_mul(u, STABLE_PI), -STABLE_PI_2); }
// W = expon.rvs() from u in (0, 1]: -log(u) * 1 + 0
ELFI_HD double stable_expon(double u) { return leaf_add(leaf_mul(-stable_log(u), 1.0), 0.0); }

// _rvs_Z1 of one (TH, W)
ELFI_HD double stable_z1(const StableRow& r, double TH, double W) {
    const double aTH = leaf_mul(r.alpha, TH);
    const double cosTH = stable_cos(TH), tanTH = stable_tan(TH);
    if (r.branch == STABLE_ALPHA1) {
        const double bTH = leaf_mul(r.beta, TH);
        const double h = leaf_add(STABLE_PI_2, bTH);
        const double lg = stable_log(gnk_div(leaf_mul(leaf_mul(STABLE_PI_2, W), cosTH), h));
        return leaf_mul(2.0 / STABLE_PI, leaf_sub(leaf_mul(h, tanTH), leaf_mul(r.beta, lg)));
    }
    const double sin_a = stable_sin(aTH), cos_a = stable_cos(aTH);
    double den, num;
    if (r.branch == STABLE_BETA0) {
        den = leaf_add(gnk_div(cosTH, stable_tan(aTH)), stable_sin(TH));
        num = leaf_add(cos_a, leaf_mul(sin_a, tanTH));
    } else {
        den = leaf_add(gnk_div(cosTH, stable_tan(leaf_mul(r.alpha, leaf_add(r.th0, TH)))),
                       stable_sin(TH));
        num = leaf_sub(leaf_add(cos_a, leaf_mul(sin_a, tanTH)),
                       leaf_mul(r.val0, leaf_sub(sin_a, leaf_mul(cos_a, tanTH))));
    }
    return leaf_mul(gnk_div(W, den), stable_pow(gnk_div(num, W), r.inv_alpha));
}

// levy_stable(alpha, beta, loc, scale).rvs of one (TH, W), S1 or S0 as r was made
ELFI_HD double stable_draw(const StableRow& r, double TH, double W) {
    double x = leaf_add(leaf_mul(stable_z1(r, TH, W), r.scale), r.loc);
    if (r.branch == STABLE_ALPHA1) x = leaf_add(x, r.shift1);
    if (r.s0) x = leaf_sub(x, r.shift0);
    return x;
}

}  // namespace elfi
