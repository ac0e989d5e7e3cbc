// gmterm.cuh -- one term of the Gaussian-mixture density of smc.cu: 2^(-nt) for the scaled,
// whitened squared distance nt with the component's log2-weight folded in (gm_pdf_kernel and
// gm_pdf_generic_kernel).  Compiles for the host as well: tests/harness/gmterm_harness.cpp calls
// the same function that the kernels inline, and tests/test_gm_formula_host.py checks it against
// mpmath.
//
// 2^(-nt): k = rint(-nt) through the 2^52 trick (no 64-bit conversions, which run on the slow XU
// pipe), f = -nt - k in [-.5, .5] (exact), 2^f by the degree-6 minimax polynomial (relative error
// < 1.9e-9, Remez on [-.5, .5]), scaled by 2^k through the exponent field; nt > 1020 flushes to 0
// (and so does a zero weight, whose nt is +inf; a NaN nt fails the compare and gives 0 too).
#pragma once

#include "hd.cuh"

#if !defined(__CUDA_ARCH__)
#include <math.h>
#include <string.h>
#include <stdint.h>
#endif

namespace elfi {

#if defined(__CUDA_ARCH__)
__device__ __forceinline__ int gm_lo(double v) { return __double2loint(v); }
__device__ __forceinline__ int gm_hi(double v) { return __double2hiint(v); }
__device__ __forceinline__ double gm_hilo(int hi, int lo) { return __hiloint2double(hi, lo); }
#else
inline int gm_lo(double v) {
    uint64_t b;
    memcpy(&b, &v, 8);
    return int(uint32_t(b));
}
inline int gm_hi(double v) {
    uint64_t b;
    memcpy(&b, &v, 8);
    return int(uint32_t(b >> 32));
}
inline double gm_hilo(int hi, int lo) {
    const uint64_t b = (uint64_t(uint32_t(hi)) << 32) | uint64_t(uint32_t(lo));
    double v;
    memcpy(&v, &b, 8);
    return v;
}
#endif

ELFI_HD double exp2_neg(double nt) {
    const double magic = 6755399441055744.0;  // 1.5 * 2^52
    const double tm = magic - nt;
    const double kd = tm - magic;             // rint(-nt)
    const double f = -nt - kd;
    double pz = 1.5345812158740182e-04;
    pz = fma(pz, f, 1.3399931209474140e-03);
    pz = fma(pz, f, 9.6184889565227916e-03);
    pz = fma(pz, f, 5.5503287769976638e-02);
    pz = fma(pz, f, 2.4022646890639572e-01);
    pz = fma(pz, f, 6.9314720573725268e-01);
    pz = fma(pz, f, 1.0000000005541663e+00);
    const int k = gm_lo(tm);                  // low word of (magic - nt) holds rint(-nt)
    const int hi = gm_hi(pz) + (k << 20);
    const double r = gm_hilo(hi, gm_lo(pz));
    return (nt <= 1020.0) ? r : 0.0;
}

}  // namespace elfi
