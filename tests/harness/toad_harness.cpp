// Host build of elfi_b200/csrc/toad.cuh (test infrastructure, see tests/test_toad_host.py).
#include <cstdint>

#include "../../elfi_b200/csrc/toad.cuh"

// out[0 .. n_p - 1]: the p quantiles of the sorted kept set v (n >= 1), out[n_p]: its median as
// nanmedian gives it for n_rows displacement rows; before nan_to_num
extern "C" void harness_toad_quantiles(const double* v, int32_t n, int32_t n_rows, int32_t n_p,
                                       const double* p, double* out) {
    for (int j = 0; j < n_p; ++j) {
        const elfi::ToadPick pk = elfi::toad_quantile_pick(n, p[j]);
        out[j] = elfi::gnk_lerp(v[pk.lo], v[pk.hi], pk.t);
    }
    int lo, hi;
    elfi::toad_median_picks(n, lo, hi);
    out[n_p] = elfi::toad_median(v[lo], v[hi], n, n_rows);
}

// out[i] = nan_to_num(log_gap(lo[i], hi[i])) and raw[i] = nan_to_num(x[i])
extern "C" void harness_toad_post(const double* lo, const double* hi, const double* x, int64_t n,
                                  double* out, double* raw) {
    for (int64_t i = 0; i < n; ++i) {
        out[i] = elfi::toad_nan_to_num(elfi::toad_log_gap(lo[i], hi[i]));
        raw[i] = elfi::toad_nan_to_num(x[i]);
    }
}

// out[i] = the levy_stable step of (alpha[i], gamma[i]) from uniforms u[i] (TH) and v[i] (W)
extern "C" void harness_toad_step(const double* alpha, const double* gamma, const double* u,
                                  const double* v, int64_t n, double* out) {
    for (int64_t i = 0; i < n; ++i)
        out[i] = elfi::toad_stable_step(alpha[i], gamma[i], elfi::toad_theta(u[i]),
                                        elfi::toad_expon(v[i]));
}

// out[i] = refuge day of word w[i] below d[i]
extern "C" void harness_toad_refuge(const uint64_t* w, const int32_t* d, int64_t n, int32_t* out) {
    for (int64_t i = 0; i < n; ++i) out[i] = elfi::toad_refuge_day(w[i], d[i]);
}

extern "C" double harness_toad_floor() { return elfi::TOAD_GAP_FLOOR; }
