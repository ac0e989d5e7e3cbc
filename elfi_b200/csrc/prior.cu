// prior.cu -- draws and joint log densities of stock scipy.stats priors (uniform, norm, truncnorm,
// expon, gamma, beta) for the throughput mode: the generic device fast path of ModelPrior
// (elfi/model/extensions.py:120-245) for models whose priors are independent and have constant
// parameters.  The table format and the per-kind arithmetic are in priors.cuh.
//
// prior_rvs_kernel: one thread per row; the value of row i is a pure function of
// (seed, offset + i), whatever the sharding, from Philox blocks (row, row >> 32, block, SALT_PRIOR):
//   uniform    block 0: u = u01(x, y);  loc + scale u
//   norm       block 0: z = first normal of Box-Muller (boxmuller.cuh);  loc + scale z
//   truncnorm  block 0: u = u01(x, y);  loc + scale sign clamp(Phi^-1(cdf_lo + u cdf_w), lo, hi),
//              mirrored when a > 0 exactly as prior_gauss_kernel draws (simulate.cu)
//   expon      block 0: u = u01(x, y);  loc - scale log(u)
//   gamma      Marsaglia-Tsang: trial t = 0, 1, .. of component g (0 for gamma and for beta's X,
//              1 for beta's Y) takes z = first normal of block (g << 16) | 2t and
//              u = u01(x, y), w = u01(z, w) of block (g << 16) | (2t + 1); the first accepted trial
//              gives G = d v, times w^(1/a) when a < 1 (G(a + 1) u^(1/a));  loc + scale G
//   beta       X = G(a) of component 0, Y = G(b) of component 1;  loc + scale X / (X + Y)
// At most PRIOR_MAX_TRIALS = 64 trials per component (include/elfi_b200.h says what the bound
// returns; for every valid shape a trial is rejected with probability below 0.05).
// The draw is fma(scale, y, loc) (loc + scale y, one rounding) with the table's loc and scale, or
// per row with loc[i] / scale[i] when those vectors are given (a conditional prior): y and its
// stream do not depend on them.  A per-row scale < 0 or NaN gives NaN (priors.cuh).
#include "boxmuller.cuh"
#include "common.cuh"
#include "philox.cuh"
#include "priors.cuh"

namespace elfi {

constexpr uint32_t SALT_PRIOR = 0x50524f52u;   // "PROR"

// G(s) of component g: d v of the first accepted trial (times w^(1/s) for s < 1); d (times 1) when
// all PRIOR_MAX_TRIALS trials are rejected
__device__ __forceinline__ double gamma_component(const Philox& ph, uint32_t r0, uint32_t r1,
                                                  uint32_t g, double d, double c, double inv_a) {
    double v = 1.0, w = 1.0;
    for (uint32_t t = 0; t < uint32_t(PRIOR_MAX_TRIALS); ++t) {
        const uint32_t blk = (g << 16) | (2u * t);
        double z, z1;
        normal2(ph(r0, r1, blk, SALT_PRIOR), z, z1);
        const uint4 q = ph(r0, r1, blk + 1u, SALT_PRIOR);
        double vt, margin;
        if (prior_mt_accept(d, c, z, u01(q.x, q.y), &vt, &margin)) {
            v = vt;
            w = u01(q.z, q.w);
            break;
        }
    }
    const double x = d * v;
    return inv_a > 0.0 ? x * pow(w, inv_a) : x;
}

__global__ void __launch_bounds__(256)
prior_rvs_kernel(int64_t B, uint64_t seed, uint64_t offset, const PriorEntry e,
                 const double* __restrict__ loc, const double* __restrict__ scale,
                 double* __restrict__ out) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= B) return;
    const Philox ph(seed);
    const uint64_t row = offset + uint64_t(i);
    const uint32_t r0 = uint32_t(row), r1 = uint32_t(row >> 32);
    double y;
    if (e.kind == PRIOR_GAMMA) {
        y = gamma_component(ph, r0, r1, 0u, e.d[0], e.c[0], e.inv_a[0]);
    } else if (e.kind == PRIOR_BETA) {
        const double gx = gamma_component(ph, r0, r1, 0u, e.d[0], e.c[0], e.inv_a[0]);
        const double gy = gamma_component(ph, r0, r1, 1u, e.d[1], e.c[1], e.inv_a[1]);
        y = gx / (gx + gy);
    } else {
        const uint4 r = ph(r0, r1, 0u, SALT_PRIOR);
        const double u = u01(r.x, r.y);
        if (e.kind == PRIOR_UNIFORM) {
            y = u;
        } else if (e.kind == PRIOR_NORM) {
            double z1;
            normal2(r, y, z1);
        } else if (e.kind == PRIOR_TRUNCNORM) {
            const double t = normcdfinv(e.t_cdf_lo + u * e.t_cdf_w);
            y = e.t_sign * fmin(fmax(t, e.t_lo), e.t_hi);
        } else {
            y = -log(u);                                     // expon
        }
    }
    const double l = loc ? loc[i] : e.loc;
    const double c = scale ? scale[i] : e.scale;
    out[i] = (c >= 0.0) ? fma(c, y, l) : NAN;
}

__global__ void __launch_bounds__(256)
prior_logpdf_kernel(const double* __restrict__ x, int64_t ld, int64_t B, int p,
                    const PriorTable tab, double* __restrict__ out) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= B) return;
    const double* row = x + i * ld;
    const auto col = [&](int j) { return row[j]; };
    double s = 0.0;
    for (int a = 0; a < p; ++a) s += prior_logpdf1(tab.e[a], row[a], col);
    out[i] = s;
}

// the table of p parameters from 5 or 7 words each
static int prior_table_from_host(const char* what, const double* spec_host, int p, int words,
                                 PriorTable* tab) {
    memset(tab, 0, sizeof(*tab));
    for (int a = 0; a < p; ++a) {
        char why[200];
        const double* s = spec_host + words * a;
        const bool ok = words == PRIOR_COND_SPEC_WORDS
                            ? prior_entry_from_spec7(s, a, p, &tab->e[a], why, sizeof(why))
                            : prior_entry_from_spec(s, &tab->e[a], why, sizeof(why));
        ELFI_REQUIRE(ok, "%s: prior parameter %d: %s", what, a, why);
    }
    return ELFI_B200_OK;
}

static int prior_rvs_launch(elfi_b200_ctx* ctx, const double* spec_host, int64_t B, uint64_t seed,
                            uint64_t offset, const double* loc, const double* scale, double* out,
                            void* stream_) {
    ELFI_REQUIRE(ctx && spec_host && B >= 0 && (B == 0 || out), "prior_rvs: bad argument");
    PriorEntry e;
    char why[160];
    ELFI_REQUIRE(prior_entry_from_words(spec_host, loc ? 0 : -1, scale ? 0 : -1, &e, why, sizeof(why)),
                 "prior_rvs: prior parameter 0: %s", why);
    if (B == 0) return ELFI_B200_OK;
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        prior_rvs_kernel<<<unsigned((B + 255) / 256), 256, 0, stream>>>(B, seed, offset, e, loc,
                                                                        scale, out);
        return ELFI_B200_OK;
    });
}

static int prior_logpdf_launch(elfi_b200_ctx* ctx, const double* x, int64_t ldx, int64_t B,
                               int64_t p, const double* spec_host, int words, double* out,
                               void* stream_) {
    ELFI_REQUIRE(ctx && spec_host && B >= 0 && (B == 0 || (x && out)), "prior_logpdf: bad argument");
    ELFI_REQUIRE(p >= 1 && p <= PRIOR_MAX_PARAMS && ldx >= p, "prior_logpdf: bad shape (1 <= p <= 16)");
    PriorTable tab;
    const int rc = prior_table_from_host("prior_logpdf", spec_host, int(p), words, &tab);
    if (rc != ELFI_B200_OK) return rc;
    if (B == 0) return ELFI_B200_OK;
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        prior_logpdf_kernel<<<unsigned((B + 255) / 256), 256, 0, stream>>>(x, ldx, B, int(p), tab,
                                                                           out);
        return ELFI_B200_OK;
    });
}

}  // namespace elfi

extern "C" {

int elfi_b200_prior_rvs_f64(elfi_b200_ctx* ctx, const double* spec_host, int64_t B, uint64_t seed,
                            uint64_t offset, double* out, void* stream_) {
    return elfi::prior_rvs_launch(ctx, spec_host, B, seed, offset, nullptr, nullptr, out, stream_);
}

int elfi_b200_prior_rvs_cond_f64(elfi_b200_ctx* ctx, const double* spec_host, int64_t B,
                                 uint64_t seed, uint64_t offset, const double* loc,
                                 const double* scale, double* out, void* stream_) {
    return elfi::prior_rvs_launch(ctx, spec_host, B, seed, offset, loc, scale, out, stream_);
}

int elfi_b200_prior_logpdf_f64(elfi_b200_ctx* ctx, const double* x, int64_t ldx, int64_t B, int64_t p,
                               const double* spec_host, double* out, void* stream_) {
    return elfi::prior_logpdf_launch(ctx, x, ldx, B, p, spec_host, elfi::PRIOR_SPEC_WORDS, out,
                                     stream_);
}

int elfi_b200_prior_logpdf_cond_f64(elfi_b200_ctx* ctx, const double* x, int64_t ldx, int64_t B,
                                    int64_t p, const double* spec_host, double* out, void* stream_) {
    return elfi::prior_logpdf_launch(ctx, x, ldx, B, p, spec_host, elfi::PRIOR_COND_SPEC_WORDS, out,
                                     stream_);
}

}  // extern "C"
