// Host build of the conditional priors of elfi_b200/csrc/priors.cuh (test infrastructure, see
// tests/test_conditional_priors_host.py).
#include <cstdint>

#include "../../elfi_b200/csrc/priors.cuh"

// spec: p x 7 table; x: n x p rows; out: n joint log densities.  Returns -1 - (index of the first
// invalid parameter) with its reason in why, or 0.
extern "C" int harness_prior_logpdf_cond(const double* spec, int64_t p, const double* x, int64_t n,
                                         double* out, char* why, int64_t why_len) {
    elfi::PriorTable tab;
    for (int64_t a = 0; a < p; ++a)
        if (!elfi::prior_entry_from_spec7(spec + 7 * a, int(a), int(p), &tab.e[a], why,
                                          size_t(why_len)))
            return int(-1 - a);
    for (int64_t i = 0; i < n; ++i) out[i] = elfi::prior_joint_logpdf(tab.e, x + i * p, int(p));
    return 0;
}
