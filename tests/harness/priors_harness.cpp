// Host build of elfi_b200/csrc/priors.cuh (test infrastructure, see tests/test_priors_host.py).
#include <cstdint>

#include "../../elfi_b200/csrc/priors.cuh"

// spec: p x 5 table; x: n x p rows; out: n joint log densities.  Returns -1 - (index of the first
// invalid parameter) with its reason in why, or 0.
extern "C" int harness_prior_logpdf(const double* spec, int64_t p, const double* x, int64_t n,
                                    double* out, char* why, int64_t why_len) {
    elfi::PriorTable tab;
    for (int64_t a = 0; a < p; ++a)
        if (!elfi::prior_entry_from_spec(spec + 5 * a, &tab.e[a], why, size_t(why_len)))
            return int(-1 - a);
    for (int64_t i = 0; i < n; ++i) out[i] = elfi::prior_joint_logpdf(tab.e, x + i * p, int(p));
    return 0;
}

// Marsaglia-Tsang decisions: accept[i], v[i] (when accepted) and margin[i] of trial (z[i], u[i])
extern "C" void harness_mt_accept(double d, double c, const double* z, const double* u, int64_t n,
                                  int32_t* accept, double* v, double* margin) {
    for (int64_t i = 0; i < n; ++i) {
        double vt = 0.0;
        accept[i] = elfi::prior_mt_accept(d, c, z[i], u[i], &vt, &margin[i]) ? 1 : 0;
        v[i] = vt;
    }
}

// the constants of one entry: [log_scale, lognorm, t_lo, t_hi, t_sign, t_cdf_lo, t_cdf_w,
// d0, c0, inv_a0, d1, c1, inv_a1]
extern "C" int harness_prior_entry(const double* spec, double* out, char* why, int64_t why_len) {
    elfi::PriorEntry e;
    if (!elfi::prior_entry_from_spec(spec, &e, why, size_t(why_len))) return -1;
    const double v[13] = {e.log_scale, e.lognorm, e.t_lo, e.t_hi, e.t_sign, e.t_cdf_lo, e.t_cdf_w,
                          e.d[0], e.c[0], e.inv_a[0], e.d[1], e.c[1], e.inv_a[1]};
    for (int k = 0; k < 13; ++k) out[k] = v[k];
    return 0;
}
