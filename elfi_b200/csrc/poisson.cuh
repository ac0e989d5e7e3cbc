// poisson.cuh -- Poisson draws of the throughput mode from Philox words (ricker.cu), and the log
// probability mass function they test against.  Compiles for the host as well
// (tests/harness/poisson_harness.cpp checks the log-pmf against mpmath and the accept / reject
// decisions against the NumPy replay tests/ricker_replay.py).
//
// poisson_draw(lam, words) with words(j) the j-th Philox block of the draw (j < POISSON_MAX_TRIALS):
//   lam == 0            0
//   lam < 0, NaN, or lam > POISSON_LAM_MAX (NumPy's limit; NumPy raises for all three)   NaN
//   0 < lam < 10        inversion from u = u01(x, y) of block 0: the smallest k with u <= F(k), the
//                       CDF summed term by term (p_0 = exp(-lam), p_k = p_{k-1} lam / k).  The search
//                       stops at k = POISSON_INV_MAX = 64 (P(X > 64) < 1e-26 for lam < 10; only a u
//                       within rounding of 1 can reach it)
//   lam >= 10           PTRS, the transformed rejection of Hoermann (1993), with NumPy's constants
//                       (random_poisson_ptrs); trial j takes U = u01(x, y) - 1/2 and V = u01(z, w)
//                       of block j.  At most POISSON_MAX_TRIALS = 32 trials (a trial is rejected
//                       with probability below 0.12); if all are rejected the draw is floor(lam).
//
// The acceptance test of PTRS compares log(V alpha / (a / us^2 + b)) with log p(k; lam).  NumPy
// evaluates the latter as -lam + k log(lam) - lgamma(k + 1): near lam = 1e14 the three terms are
// ~3e15 and cancel to ~30, an absolute error of several units.  Here it is Loader's saddle-point
// form (Loader 2000, "Fast and accurate computation of binomial probabilities"),
//   log p(k; lam) = -(stirlerr(k) + bd0(k, lam)) - log(2 pi k) / 2,
// whose terms are all small: stirlerr(k) = log k! - log(sqrt(2 pi k) (k/e)^k) < 0.09, bd0(k, lam)
// = k log(k / lam) + lam - k >= 0 is at most ~50 within 10 sd of lam, summed as Loader's series in
// v = (k - lam) / (k + lam) whenever |k - lam| < 0.1 (k + lam) (every term positive; k - lam is
// exact), and log(2 pi k) / 2 < 23.  No step subtracts two large numbers, so the absolute error
// stays near 1e-14 for every lam up to POISSON_LAM_MAX.
//
// Every product that feeds a sum is rounded on its own (no FMA contraction), so the host build,
// the device and the replay agree except where a transcendental function differs in the last bit.
#pragma once

#include <math.h>
#include <stdint.h>

#include "philox.cuh"

#include "hd.cuh"
#include "../../include/elfi_b200.h"

namespace elfi {

constexpr double POISSON_LAM_MAX = ELFI_B200_POISSON_LAM_MAX;   // NumPy's POISSON_LAM_MAX
constexpr double POISSON_SWITCH = 10.0;                    // inversion below, PTRS at and above
constexpr int POISSON_INV_MAX = 64;
constexpr int POISSON_MAX_TRIALS = 32;
constexpr double POISSON_HALF_LOG_2PI = 0.9189385332046728;   // log(2 pi) / 2

ELFI_HD double pois_add(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
ELFI_HD double pois_sub(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dsub_rn(a, b);
#else
    return a - b;
#endif
}
ELFI_HD double pois_mul(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}

// stirlerr(n) = log(n!) - log(sqrt(2 pi n) (n / e)^n) for an integer n >= 1: exact values (to
// double precision) up to 15, the asymptotic series beyond
ELFI_HD double poisson_stirlerr(double n) {
    if (n <= 15.0) {
        switch (int(n)) {
        case 1: return 0.08106146679532726;
        case 2: return 0.0413406959554093;
        case 3: return 0.02767792568499834;
        case 4: return 0.020790672103765093;
        case 5: return 0.016644691189821193;
        case 6: return 0.013876128823070748;
        case 7: return 0.01189670994589177;
        case 8: return 0.010411265261972096;
        case 9: return 0.009255462182712733;
        case 10: return 0.00833056343336287;
        case 11: return 0.007573675487951841;
        case 12: return 0.00694284010720953;
        case 13: return 0.006408994188004207;
        case 14: return 0.0059513701127588475;
        default: return 0.005554733551962801;
        }
    }
    const double S0 = 1.0 / 12, S1 = 1.0 / 360, S2 = 1.0 / 1260, S3 = 1.0 / 1680, S4 = 1.0 / 1188;
    const double nn = pois_mul(n, n);
    return pois_sub(S0, pois_sub(S1, pois_sub(S2, pois_sub(S3, S4 / nn) / nn) / nn) / nn) / n;
}

// bd0(x, m) = x log(x / m) + m - x >= 0 (Loader's deviance term)
ELFI_HD double poisson_bd0(double x, double m) {
    const double dx = pois_sub(x, m);
    if (fabs(dx) < pois_mul(0.1, pois_add(x, m))) {
        double v = dx / pois_add(x, m);
        double s = pois_mul(dx, v);
        double ej = pois_mul(pois_mul(2.0, x), v);
        v = pois_mul(v, v);
        for (int j = 1; j < 32; ++j) {             // |v| < 0.1: a term shrinks 100-fold per step
            ej = pois_mul(ej, v);
            const double s1 = pois_add(s, ej / double(2 * j + 1));
            if (s1 == s) break;
            s = s1;
        }
        return s;
    }
    return pois_add(pois_mul(x, log(x / m)), pois_sub(m, x));
}

// log p(k; lam) for an integer-valued k >= 0 and lam > 0
ELFI_HD double poisson_logpmf(double k, double lam) {
    if (k == 0.0) return -lam;
    return pois_sub(-pois_add(poisson_stirlerr(k), poisson_bd0(k, lam)),
                    pois_add(POISSON_HALF_LOG_2PI, pois_mul(0.5, log(k))));
}

// PTRS constants of a rate lam >= 10 (NumPy's random_poisson_ptrs)
struct PtrsConst {
    double b, a, log_invalpha, vr;
};

ELFI_HD PtrsConst ptrs_const(double lam) {
    PtrsConst c;
    c.b = pois_add(0.931, pois_mul(2.53, sqrt(lam)));
    c.a = pois_add(-0.059, pois_mul(0.02483, c.b));
    c.log_invalpha = log(pois_add(1.1239, 1.1328 / pois_sub(c.b, 3.4)));
    c.vr = pois_sub(0.9277, 3.6224 / pois_sub(c.b, 2.0));
    return c;
}

// One PTRS trial from U in (-1/2, 1/2] and V in (0, 1].  Returns 1 (accept *k), 0 (reject);
// *margin = |lhs - log p| of the log-pmf test when it was taken, else +inf (the other tests
// compare exactly rounded values, which the host build and the replay reproduce bit for bit).
ELFI_HD int ptrs_trial(const PtrsConst& c, double lam, double U, double V, double* k,
                       double* margin) {
    *margin = INFINITY;
    const double us = pois_sub(0.5, fabs(U));
    const double kf = floor(pois_add(pois_add(pois_mul(pois_add(pois_mul(2.0, c.a) / us, c.b), U), lam),
                                     0.43));
    *k = kf;
    if (us >= 0.07 && V <= c.vr) return 1;
    if (kf < 0.0 || (us < 0.013 && V > us)) return 0;
    const double lhs = pois_sub(pois_add(log(V), c.log_invalpha),
                                log(pois_add(c.a / pois_mul(us, us), c.b)));
    const double rhs = poisson_logpmf(kf, lam);
    *margin = fabs(pois_sub(lhs, rhs));
    return lhs <= rhs ? 1 : 0;
}

// A draw: the count k, the blocks used (0 for lam == 0 and the NaN results) and the smallest
// decision margin, relative to the compared values for inversion (|u - F| / F) and absolute for
// PTRS's log-pmf test (+inf when no decision was inexact).
struct PoissonDraw {
    double k;
    int trials;
    double margin;
};

// Words: j -> PhiloxWords, the j-th block of this draw
template <class Words>
ELFI_HD PoissonDraw poisson_draw(double lam, const Words& words) {
    PoissonDraw d{0.0, 0, INFINITY};
    if (!(lam >= 0.0) || lam > POISSON_LAM_MAX) {
        d.k = NAN;
        return d;
    }
    if (lam == 0.0) return d;
    if (lam < POISSON_SWITCH) {
        const PhiloxWords w = words(0);
        const double u = u01(w.x, w.y);
        double p = exp(-lam), F = p;
        int k = 0;
        for (; k < POISSON_INV_MAX; ++k) {
            d.margin = fmin(d.margin, fabs(pois_sub(u, F)) / F);
            if (u <= F) break;
            p = pois_mul(p, lam) / double(k + 1);
            F = pois_add(F, p);
        }
        d.k = double(k);
        d.trials = 1;
        return d;
    }
    const PtrsConst c = ptrs_const(lam);
    d.k = floor(lam);
    d.trials = POISSON_MAX_TRIALS;
    for (int j = 0; j < POISSON_MAX_TRIALS; ++j) {
        const PhiloxWords w = words(j);
        double k, mg;
        const int acc = ptrs_trial(c, lam, pois_sub(u01(w.x, w.y), 0.5), u01(w.z, w.w), &k, &mg);
        d.margin = fmin(d.margin, mg);
        if (acc) {
            d.k = k;
            d.trials = j + 1;
            break;
        }
    }
    return d;
}

}  // namespace elfi
