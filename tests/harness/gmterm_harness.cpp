// Host build of elfi_b200/csrc/gmterm.cuh: the 2^(-nt) term of the mixture-density kernels
// (smc.cu), exported over a flat array so that tests/test_gm_formula_host.py can check the
// shipped polynomial, range reduction and flush against mpmath.  Test infrastructure only.
#include <cstdint>

#include "../../elfi_b200/csrc/gmterm.cuh"

extern "C" void harness_exp2_neg(const double* nt, int64_t n, double* out) {
    for (int64_t i = 0; i < n; ++i) out[i] = elfi::exp2_neg(nt[i]);
}
