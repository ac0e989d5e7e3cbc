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
    out[i] = e.loc + e.scale * y;
}

__global__ void __launch_bounds__(256)
prior_logpdf_kernel(const double* __restrict__ x, int64_t ld, int64_t B, int p,
                    const PriorTable tab, double* __restrict__ out) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= B) return;
    double s = 0.0;
    for (int a = 0; a < p; ++a) s += prior_logpdf1(tab.e[a], x[i * ld + a]);
    out[i] = s;
}

}  // namespace elfi

extern "C" {

int elfi_b200_prior_rvs_f64(elfi_b200_ctx* ctx, const double* spec_host, int64_t B, uint64_t seed,
                            uint64_t offset, double* out, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && spec_host && B >= 0 && (B == 0 || out), "prior_rvs: bad argument");
    PriorEntry e;
    char why[160];
    ELFI_REQUIRE(prior_entry_from_spec(spec_host, &e, why, sizeof(why)),
                 "prior_rvs: prior parameter 0: %s", why);
    if (B == 0) return ELFI_B200_OK;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    ELFI_CUDA_OK(cudaSetDevice(ctx->device));
    prior_rvs_kernel<<<unsigned((B + 255) / 256), 256, 0, stream>>>(B, seed, offset, e, out);
    ELFI_CUDA_OK(cudaGetLastError());
    return ELFI_B200_OK;
}

int elfi_b200_prior_logpdf_f64(elfi_b200_ctx* ctx, const double* x, int64_t ldx, int64_t B, int64_t p,
                               const double* spec_host, double* out, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && spec_host && B >= 0 && (B == 0 || (x && out)), "prior_logpdf: bad argument");
    ELFI_REQUIRE(p >= 1 && p <= PRIOR_MAX_PARAMS && ldx >= p, "prior_logpdf: bad shape (1 <= p <= 16)");
    PriorTable tab;
    memset(&tab, 0, sizeof(tab));
    for (int a = 0; a < p; ++a) {
        char why[160];
        ELFI_REQUIRE(prior_entry_from_spec(spec_host + PRIOR_SPEC_WORDS * a, &tab.e[a], why, sizeof(why)),
                     "prior_logpdf: prior parameter %d: %s", a, why);
    }
    if (B == 0) return ELFI_B200_OK;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    ELFI_CUDA_OK(cudaSetDevice(ctx->device));
    prior_logpdf_kernel<<<unsigned((B + 255) / 256), 256, 0, stream>>>(x, ldx, B, int(p), tab, out);
    ELFI_CUDA_OK(cudaGetLastError());
    return ELFI_B200_OK;
}

}  // extern "C"
