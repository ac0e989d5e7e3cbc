// priors.cuh -- stock scipy.stats priors of the throughput mode: the per-parameter table entry, the
// host code that fills it from scipy's positional parameters, and the plain fp64 arithmetic shared
// by the device kernels (prior.cu, the support-3 proposals of simulate.cu) and the host build of
// tests/harness/priors_harness.cpp: the standardised log density of each kind, its support test and
// the Marsaglia-Tsang acceptance test.
//
// A parameter is specified by five doubles [kind, p0, p1, p2, p3], scipy's positional parameters
// with loc / scale filled in (Python's elfi_b200.priors does that):
//   kind 0 uniform    (loc, scale)          support [loc, loc + scale]
//   kind 1 norm       (loc, scale)          R
//   kind 2 truncnorm  (a, b, loc, scale)    [loc + a scale, loc + b scale]
//   kind 3 expon      (loc, scale)          [loc, inf)
//   kind 4 gamma      (a, loc, scale)       [loc, inf)
//   kind 5 beta       (a, b, loc, scale)    [loc, loc + scale]
// The log density is scipy.stats.<kind>.logpdf: y = (x - loc) / scale, -inf where y is outside the
// closed support, else the standardised log density of y minus log(scale) -- with scipy's values
// on the support edges (xlogy / xlog1py: +inf for gamma a < 1 or beta a < 1 at y = 0, finite for
// a = 1, -inf for a > 1; the same for beta's b at y = 1).  NaN in, NaN out.
//
// Conditional loc / scale.  An entry's loc and scale may instead come from another column of the
// same row (loc_src, scale_src: -1 the table's constant, j the column j != the parameter itself),
// as in a hierarchical model where t2 ~ U(t1, t1 + 10).  The 7-word form [kind, p0, p1, p2, p3,
// loc_src, scale_src] carries them; a sourced word among the first five is a placeholder and is
// not validated.  Shape parameters always are constants.  The draw loc + scale y keeps y's stream,
// so only the affine step and the density's (x - loc) / scale and log(scale) become per-row.
// Per-row rule (SciPy 1.18.1's):
//   logpdf: a scale that is not > 0, or NaN, gives NaN; a NaN loc gives NaN; an infinite scale
//           gives y = 0 (or NaN for an infinite x - loc) and so -inf for uniform (-log(inf));
//   rvs:    a scale of 0 gives loc; a NaN loc gives NaN; a scale < 0 or NaN gives NaN (SciPy raises).
// A sourced scale takes its log on the device; a constant one keeps the host-computed log_scale,
// so with every source at -1 the densities are the bits of the 5-word table.
#pragma once

#include <math.h>
#include <stdint.h>
#include <stdio.h>

#include "hd.cuh"
#include "../../include/elfi_b200.h"

namespace elfi {

enum PriorKind { PRIOR_UNIFORM = 0, PRIOR_NORM = 1, PRIOR_TRUNCNORM = 2, PRIOR_EXPON = 3,
                 PRIOR_GAMMA = 4, PRIOR_BETA = 5 };
// [kind, p0, p1, p2, p3] per parameter
constexpr int PRIOR_SPEC_WORDS = ELFI_B200_PRIOR_SPEC_WORDS;
// [kind, p0, p1, p2, p3, loc_src, scale_src]
constexpr int PRIOR_COND_SPEC_WORDS = ELFI_B200_PRIOR_COND_SPEC_WORDS;
constexpr int PRIOR_MAX_PARAMS = ELFI_B200_MAX_PRIOR_PARAMS;
constexpr int PRIOR_MAX_TRIALS = 64;     // Marsaglia-Tsang trials per gamma component
constexpr double PRIOR_NORM_LOGC = 0.91893853320467274178;   // log(sqrt(2 pi))

struct PriorEntry {
    int kind;
    int loc_src, scale_src;   // -1: loc / scale are the constants below; j: column j of the row
    double loc, scale, log_scale;
    double a, b;           // shapes: truncnorm's bounds, gamma's a, beta's a and b
    double lognorm;        // truncnorm: log of the mass in [a, b]; gamma: lgamma(a); beta: betaln(a, b)
    // truncnorm draws: inverse CDF on [lo, hi] = [a, b], or on the mirror image [-b, -a] with
    // sign = -1 when a > 0 (the upper tail, where Phi(a) rounds to 1); cdf_w = Phi(hi) - Phi(lo)
    double t_lo, t_hi, t_sign, t_cdf_lo, t_cdf_w;
    // Marsaglia-Tsang constants of gamma component g (0: a, 1: beta's b): G(s) for s >= 1 is
    // d v with d = s - 1/3; for s < 1 it is G(s + 1) u^(1/s), then inv_a = 1/s (else 0)
    double d[2], c[2], inv_a[2];
};

struct PriorTable { PriorEntry e[PRIOR_MAX_PARAMS]; };

// scipy.special.xlogy / xlog1py: 0 when the factor is 0 (and y is not NaN)
ELFI_HD double prior_xlogy(double f, double y) {
    return (f == 0.0 && y == y) ? 0.0 : f * log(y);
}

ELFI_HD double prior_xlog1py(double f, double y) {
    return (f == 0.0 && y == y) ? 0.0 : f * log1p(y);
}

// closed support of the standardised variable y
ELFI_HD bool prior_in_support(const PriorEntry& e, double y) {
    switch (e.kind) {
    case PRIOR_NORM: return y == y;
    case PRIOR_TRUNCNORM: return y >= e.a && y <= e.b;
    case PRIOR_EXPON:
    case PRIOR_GAMMA: return y >= 0.0;
    default: return y >= 0.0 && y <= 1.0;          // uniform, beta
    }
}

// standardised log density at y inside the support (scipy's _logpdf of the kind)
ELFI_HD double prior_std_logpdf(const PriorEntry& e, double y) {
    switch (e.kind) {
    case PRIOR_UNIFORM: return 0.0;
    case PRIOR_NORM: return -y * y / 2.0 - PRIOR_NORM_LOGC;
    case PRIOR_TRUNCNORM: return (-y * y / 2.0 - PRIOR_NORM_LOGC) - e.lognorm;
    case PRIOR_EXPON: return -y;
    case PRIOR_GAMMA: return (prior_xlogy(e.a - 1.0, y) - y) - e.lognorm;
    default: return (prior_xlog1py(e.b - 1.0, -y) + prior_xlogy(e.a - 1.0, y)) - e.lognorm;
    }
}

// scipy.stats.<kind>.logpdf(x, *params) of a parameter of the row whose column j is col(j)
// (read only for a sourced loc or scale).  COND = false compiles the sources out, for tables
// known to have none.
template <bool COND = true, class Col>
ELFI_HD double prior_logpdf1(const PriorEntry& e, double x, const Col& col) {
    const double loc = (COND && e.loc_src >= 0) ? col(e.loc_src) : e.loc;
    double scale = e.scale, log_scale = e.log_scale;
    if (COND && e.scale_src >= 0) {
        scale = col(e.scale_src);
        if (!(scale > 0.0)) return NAN;
        log_scale = log(scale);
    }
    const double y = (x - loc) / scale;
    if (y != y) return y;
    if (!prior_in_support(e, y)) return -INFINITY;
    return prior_std_logpdf(e, y) - log_scale;
}

// x[src] of a row held in a local array: an unrolled select over PMAX, so that x[] can stay in
// registers (an indexed load would put it on the stack)
template <int PMAX>
ELFI_HD double prior_pick(const double* x, int src) {
    double v = 0.0;
#pragma unroll
    for (int b = 0; b < PMAX; ++b)
        if (b == src) v = x[b];
    return v;
}

// joint log density of p <= PMAX parameters: the terms summed left to right (the loop is
// unrolled over PMAX so that a caller's x[] can live in registers)
template <int PMAX = PRIOR_MAX_PARAMS, bool COND = true>
ELFI_HD double prior_joint_logpdf(const PriorEntry* e, const double* x, int p) {
    double s = 0.0;
    const auto col = [&](int j) { return prior_pick<PMAX>(x, j); };
#pragma unroll
    for (int a = 0; a < PMAX; ++a)
        if (a < p) s += prior_logpdf1<COND>(e[a], x[a], col);
    return s;
}

// One Marsaglia-Tsang trial of G(d + 1/3) from a standard normal z and a uniform u in (0, 1]:
// accepted iff 1 + c z > 0 and log u < z^2 / 2 + d - d v + d log v with v = (1 + c z)^3; the
// draw is then d v.  *margin: the distance of log u from the bound (for replays that exclude
// knife-edge decisions), or +inf when 1 + c z <= 0.
ELFI_HD bool prior_mt_accept(double d, double c, double z, double u, double* v,
                             double* margin) {
    const double t = 1.0 + c * z;
    if (!(t > 0.0)) {
        *margin = INFINITY;
        return false;
    }
    const double vt = t * t * t;
    const double bound = 0.5 * z * z + d - d * vt + d * log(vt);
    const double lu = log(u);
    *v = vt;
    *margin = fabs(bound - lu);
    return lu < bound;
}

// ---- host: the table entry from [kind, p0, p1, p2, p3] ------------------------------------------
// Returns false and writes the reason to why[n] for invalid parameters.
inline double prior_log_gauss_mass(double a, double b) {
    const double r = 0.70710678118654752440;
    if (b <= 0.0) return log(0.5 * erfc(-b * r) - 0.5 * erfc(-a * r));
    if (a > 0.0) return log(0.5 * erfc(a * r) - 0.5 * erfc(b * r));   // the upper tail, mirrored
    return log1p(-0.5 * erfc(-a * r) - 0.5 * erfc(b * r));           // 1 - Phi(a) - Phi(-b)
}

inline void prior_gamma_constants(double s, double* d, double* c, double* inv_a) {
    *inv_a = s < 1.0 ? 1.0 / s : 0.0;
    *d = (s < 1.0 ? s + 1.0 : s) - 1.0 / 3.0;
    *c = 1.0 / sqrt(9.0 * *d);
}

// loc_src / scale_src: -1 or the column the row supplies it from (checked by the caller); a sourced
// loc or scale word of s is not read
inline bool prior_entry_from_words(const double* s, int loc_src, int scale_src, PriorEntry* e,
                                   char* why, size_t n) {
    const double k = s[0];
    *e = PriorEntry();
    e->loc_src = loc_src;
    e->scale_src = scale_src;
    if (!(k == 0.0 || k == 1.0 || k == 2.0 || k == 3.0 || k == 4.0 || k == 5.0)) {
        snprintf(why, n, "unknown kind %g (0 uniform, 1 norm, 2 truncnorm, 3 expon, 4 gamma, 5 beta)", k);
        return false;
    }
    e->kind = int(k);
    const int nshape = (e->kind == PRIOR_TRUNCNORM || e->kind == PRIOR_BETA) ? 2 :
                       (e->kind == PRIOR_GAMMA ? 1 : 0);
    e->a = nshape >= 1 ? s[1] : 0.0;
    e->b = nshape >= 2 ? s[2] : 0.0;
    e->loc = loc_src < 0 ? s[1 + nshape] : 0.0;
    e->scale = scale_src < 0 ? s[2 + nshape] : 1.0;
    if (!(e->scale > 0.0) || !isfinite(e->scale) || !isfinite(e->loc)) {
        snprintf(why, n, "loc must be finite and scale finite and > 0 (loc %g, scale %g)", e->loc, e->scale);
        return false;
    }
    e->log_scale = log(e->scale);
    switch (e->kind) {
    case PRIOR_TRUNCNORM: {
        if (!(e->a < e->b)) {
            snprintf(why, n, "truncnorm needs a < b (a %g, b %g)", e->a, e->b);
            return false;
        }
        e->lognorm = prior_log_gauss_mass(e->a, e->b);
        const bool mirror = e->a > 0.0;
        e->t_lo = mirror ? -e->b : e->a;
        e->t_hi = mirror ? -e->a : e->b;
        e->t_sign = mirror ? -1.0 : 1.0;
        e->t_cdf_lo = 0.5 * erfc(-e->t_lo * 0.7071067811865476);
        e->t_cdf_w = 0.5 * erfc(-e->t_hi * 0.7071067811865476) - e->t_cdf_lo;
        break;
    }
    case PRIOR_GAMMA:
        if (!(e->a > 0.0) || !isfinite(e->a)) {
            snprintf(why, n, "gamma needs a finite a > 0 (a %g)", e->a);
            return false;
        }
        e->lognorm = lgamma(e->a);
        prior_gamma_constants(e->a, &e->d[0], &e->c[0], &e->inv_a[0]);
        break;
    case PRIOR_BETA:
        if (!(e->a > 0.0) || !(e->b > 0.0) || !isfinite(e->a) || !isfinite(e->b)) {
            snprintf(why, n, "beta needs finite a > 0 and b > 0 (a %g, b %g)", e->a, e->b);
            return false;
        }
        e->lognorm = lgamma(e->a) + lgamma(e->b) - lgamma(e->a + e->b);
        prior_gamma_constants(e->a, &e->d[0], &e->c[0], &e->inv_a[0]);
        prior_gamma_constants(e->b, &e->d[1], &e->c[1], &e->inv_a[1]);
        break;
    default:
        break;
    }
    return true;
}

// the 5-word form: constant loc and scale
inline bool prior_entry_from_spec(const double* s, PriorEntry* e, char* why, size_t n) {
    return prior_entry_from_words(s, -1, -1, e, why, n);
}

// the 7-word form of parameter a of p: words 5 and 6 are loc_src and scale_src, each -1 or an
// integer column 0 <= j < p other than a
inline bool prior_entry_from_spec7(const double* s, int a, int p, PriorEntry* e, char* why,
                                   size_t n) {
    int src[2];
    for (int w = 0; w < 2; ++w) {
        const double v = s[PRIOR_SPEC_WORDS + w];
        if (!(v == -1.0 || (v >= 0.0 && v < double(p) && v == floor(v) && v != double(a)))) {
            snprintf(why, n, "%s source must be -1 or a column 0 <= j < %d other than %d (got %g)",
                     w ? "scale" : "loc", p, a, v);
            return false;
        }
        src[w] = int(v);
    }
    return prior_entry_from_words(s, src[0], src[1], e, why, n);
}

}  // namespace elfi
