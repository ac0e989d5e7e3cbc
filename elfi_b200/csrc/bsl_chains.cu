// bsl_chains.cu -- one Metropolis-Hastings step of C lock-step BSL chains in throughput mode
// (elfi/methods/inference/bsl.py: BSL's random-walk sampler, with its logit-transformed proposals
// and its Jacobian rule), so that proposals, prior densities, decisions and the chain storage stay
// on the device and the host only launches work.
//
// One CTA per chain.  Thread 0 makes the chain's decision for iteration t and draws the proposal of
// iteration t + 1; then the CTA writes the chain's b rows of the next batch's parameters.
//
// Random stream (Philox4x32-10 keyed by the sampler's seed, or by keys[c] in the keyed entry point;
// include/elfi_b200.h has the contract).  With lane l = c, or lanes[c] in the keyed entry point:
//   counter (t, l, 0, SALT_BSL):      u = u01(x, y), the uniform of chain c's decision at iteration t
//   counter (t, l, 1 + k, SALT_BSL):  z_2k, z_2k+1 (Box-Muller, boxmuller.cuh) of chain c's
//                                     proposal for iteration t, k = 0 .. ceil(p / 2) - 1
// so no value depends on C, on the other chains or on the launch shape, and the chains of several
// samplers (a Testbench's repetitions) can step in one launch.
#include "boxmuller.cuh"
#include "common.cuh"
#include "philox.cuh"
#include "priors.cuh"

namespace elfi {

constexpr uint32_t SALT_BSL = 0x4253434cu;   // "BSCL"
constexpr int BSL_THREADS = 128;
constexpr int64_t BSL_MAX_CHAINS = ELFI_B200_BSL_MAX_CHAINS;
constexpr int BSL_TRI = PRIOR_MAX_PARAMS * (PRIOR_MAX_PARAMS + 1) / 2;

// logit kinds of a parameter, by which of its bounds (a, b) are finite
enum BslBound { BSL_BOTH = 0, BSL_UPPER = 1, BSL_LOWER = 2, BSL_NONE = 3 };

struct BslStepParams {
    PriorTable prior;
    double L[BSL_TRI];                          // Cholesky factor, lower triangle row by row
    double lo[PRIOR_MAX_PARAMS], hi[PRIOR_MAX_PARAMS];
    int kind[PRIOR_MAX_PARAMS];                 // BslBound; BSL_NONE for every parameter without bounds
};

// theta -> the proposal space: log((x - a) / (b - x)), log(1 / (b - x)), log(x - a) or x
__device__ __forceinline__ double bsl_logit(int kind, double a, double b, double x) {
    switch (kind) {
    case BSL_BOTH: return log((x - a) / (b - x));
    case BSL_UPPER: return log(1.0 / (b - x));
    case BSL_LOWER: return log(x - a);
    default: return x;
    }
}

__device__ __forceinline__ double bsl_logit_back(int kind, double a, double b, double y) {
    if (kind == BSL_NONE) return y;
    const double ey = exp(y);
    switch (kind) {
    case BSL_BOTH: return a / (1.0 + ey) + b / (1.0 + (1.0 / ey));
    case BSL_UPPER: return b - (1.0 / ey);
    default: return a + ey;
    }
}

// log |d theta / d theta~| of the back transform evaluated at theta itself (the reference's rule),
// summed left to right
template <int PMAX>
__device__ __forceinline__ double bsl_jacobian(const BslStepParams& P, const double* x, int p) {
    double s = 0.0;
#pragma unroll
    for (int a = 0; a < PMAX; ++a) {
        if (a >= p) break;
        double v = 0.0;
        if (P.kind[a] == BSL_BOTH) {
            const double ey = exp(x[a]);
            v = log(P.hi[a] - P.lo[a]) - log((1.0 / ey) + 2.0 + ey);
        } else if (P.kind[a] != BSL_NONE) {
            v = x[a];
        }
        s += v;
    }
    return s;
}

template <int PMAX>
__global__ void __launch_bounds__(BSL_THREADS)
bsl_mh_step_kernel(const BslStepParams P, int p, int64_t t, int64_t n_samples, int64_t burn_in,
                   int64_t b, uint64_t seed, const uint64_t* __restrict__ keys,
                   const uint32_t* __restrict__ lanes, const double* __restrict__ loglik,
                   double* __restrict__ prop, double* __restrict__ prop_lp,
                   double* __restrict__ chains, double* __restrict__ logpost,
                   int64_t* __restrict__ n_acc, double* __restrict__ rows, int64_t ld_rows) {
    __shared__ double row[PMAX];
    const int64_t c = blockIdx.x;
    const bool next = t + 1 < n_samples;
    if (threadIdx.x == 0) {
        // NULL keys and lanes: the sampler's seed and lane c
        const Philox ph(keys ? keys[c] : seed);
        const uint32_t lane = lanes ? lanes[c] : uint32_t(c);
        double* pc = prop + c * p;
        double* state = chains + (c * n_samples + t) * p;
        double* lpost = logpost + c * n_samples + t;
        const double lp_prop = prop_lp[c];
        double s[PMAX];
#pragma unroll
        for (int a = 0; a < PMAX; ++a) s[a] = a < p ? pc[a] : 0.0;
        bool accept = true;
        double lp_new = loglik[c] + lp_prop;
        if (t > 0) {
            accept = false;
            if (isfinite(lp_prop)) {
                double prev[PMAX];
#pragma unroll
                for (int a = 0; a < PMAX; ++a) prev[a] = a < p ? state[a - p] : 0.0;
                const double res = (bsl_jacobian<PMAX>(P, s, p) - bsl_jacobian<PMAX>(P, prev, p))
                                   + (lp_new - lpost[-1]);
                const double prob = fmin(1.0, exp(fmin(700.0, fmax(-700.0, res))));
                const uint4 r = ph(uint32_t(t), lane, 0u, SALT_BSL);
                accept = u01(r.x, r.y) < prob;
            }
            if (!accept) {
#pragma unroll
                for (int a = 0; a < PMAX; ++a) s[a] = a < p ? state[a - p] : 0.0;
                lp_new = lpost[-1];
            }
        }
#pragma unroll
        for (int a = 0; a < PMAX; ++a)
            if (a < p) state[a] = s[a];
        *lpost = lp_new;
        if (accept && t >= burn_in) n_acc[c] += 1;
        if (next) {
            // the proposal of iteration t + 1: theta~ + L z in the transformed space, accumulated
            // for each parameter a over z_0 .. z_a in order
            double y[PMAX];
#pragma unroll
            for (int a = 0; a < PMAX; ++a) y[a] = a < p ? bsl_logit(P.kind[a], P.lo[a], P.hi[a], s[a]) : 0.0;
#pragma unroll
            for (int k = 0; k < PMAX; k += 2) {
                if (k >= p) break;
                double z0, z1;
                normal2(ph(uint32_t(t + 1), lane, 1u + uint32_t(k / 2), SALT_BSL), z0, z1);
#pragma unroll
                for (int a = k; a < PMAX; ++a) {
                    if (a >= p) break;
                    y[a] += P.L[a * (a + 1) / 2 + k] * z0;
                    if (a > k) y[a] += P.L[a * (a + 1) / 2 + k + 1] * z1;
                }
            }
#pragma unroll
            for (int a = 0; a < PMAX; ++a)
                if (a < p) y[a] = bsl_logit_back(P.kind[a], P.lo[a], P.hi[a], y[a]);
            const double lp = prior_joint_logpdf<PMAX, true>(P.prior.e, y, p);
            const bool inside = isfinite(lp);
#pragma unroll
            for (int a = 0; a < PMAX; ++a) {
                if (a < p) {
                    pc[a] = y[a];
                    row[a] = inside ? y[a] : s[a];
                }
            }
            prop_lp[c] = lp;
        }
    }
    if (!next) return;
    __syncthreads();
    // the chain's b rows of every column of the next batch
    for (int a = 0; a < p; ++a) {
        const double v = row[a];
        double* col = rows + a * ld_rows + c * b;
        for (int64_t i = threadIdx.x; i < b; i += BSL_THREADS) col[i] = v;
    }
}

static int bsl_mh_step_launch(elfi_b200_ctx* ctx, int64_t C, int64_t p, int64_t t,
                              int64_t n_samples, int64_t burn_in, int64_t b, uint64_t seed,
                              const uint64_t* keys, const uint32_t* lanes,
                              const double* spec_host, const double* chol_host,
                              const double* bounds_host, const double* loglik, double* prop,
                              double* prop_lp, double* chains, double* logpost, int64_t* n_acc,
                              double* rows, int64_t ld_rows, void* stream_) {
    ELFI_REQUIRE(ctx && spec_host && chol_host, "bsl_mh_step: bad argument");
    ELFI_REQUIRE(C >= 1 && C <= BSL_MAX_CHAINS, "bsl_mh_step: 1 <= C <= 2^22 chains, got %lld",
                 (long long)C);
    ELFI_REQUIRE(p >= 1 && p <= PRIOR_MAX_PARAMS, "bsl_mh_step: 1 <= p <= 16, got %lld",
                 (long long)p);
    ELFI_REQUIRE(n_samples >= 1 && n_samples <= int64_t(UINT32_MAX) && t >= 0 && t < n_samples
                     && burn_in >= 0,
                 "bsl_mh_step: need 0 <= t < n_samples < 2^32 and burn_in >= 0 (t %lld, "
                 "n_samples %lld, burn_in %lld)", (long long)t, (long long)n_samples,
                 (long long)burn_in);
    ELFI_REQUIRE(b >= 1 && C * b < (int64_t(1) << 31) && ld_rows >= C * b,
                 "bsl_mh_step: need b >= 1, C b < 2^31 and ld_rows >= C b (b %lld, ld_rows %lld)",
                 (long long)b, (long long)ld_rows);
    ELFI_REQUIRE(loglik && prop && prop_lp && chains && logpost && n_acc && rows,
                 "bsl_mh_step: bad argument (NULL device array)");
    BslStepParams P;
    memset(&P, 0, sizeof(P));
    for (int a = 0; a < int(p); ++a) {
        char why[200];
        ELFI_REQUIRE(prior_entry_from_spec7(spec_host + PRIOR_COND_SPEC_WORDS * a, a, int(p),
                                            &P.prior.e[a], why, sizeof(why)),
                     "bsl_mh_step: prior parameter %d: %s", a, why);
        for (int k = 0; k <= a; ++k) {
            const double v = chol_host[a * p + k];
            ELFI_REQUIRE(isfinite(v), "bsl_mh_step: the Cholesky factor is not finite at (%d, %d)",
                         a, k);
            P.L[a * (a + 1) / 2 + k] = v;
        }
        P.kind[a] = BSL_NONE;
        if (bounds_host) {
            const double lo = bounds_host[2 * a], hi = bounds_host[2 * a + 1];
            ELFI_REQUIRE(lo == lo && hi == hi, "bsl_mh_step: bound %d is NaN", a);
            P.lo[a] = lo;
            P.hi[a] = hi;
            P.kind[a] = (isinf(lo) ? 1 : 0) + (isinf(hi) ? 2 : 0);
        }
    }
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        with_pow2<2, PRIOR_MAX_PARAMS>(int(p), [&](auto pm) {
            bsl_mh_step_kernel<decltype(pm)::value><<<unsigned(C), BSL_THREADS, 0, stream>>>(
                P, int(p), t, n_samples, burn_in, b, seed, keys, lanes, loglik, prop, prop_lp,
                chains, logpost, n_acc, rows, ld_rows);
            return 0;
        });
        return ELFI_B200_OK;
    });
}

}  // namespace elfi

extern "C" {

int elfi_b200_bsl_mh_step_f64(elfi_b200_ctx* ctx, int64_t C, int64_t p, int64_t t,
                              int64_t n_samples, int64_t burn_in, int64_t b, uint64_t seed,
                              const double* spec_host, const double* chol_host,
                              const double* bounds_host, const double* loglik, double* prop,
                              double* prop_lp, double* chains, double* logpost, int64_t* n_acc,
                              double* rows, int64_t ld_rows, void* stream) {
    return elfi::bsl_mh_step_launch(ctx, C, p, t, n_samples, burn_in, b, seed, nullptr, nullptr,
                                    spec_host, chol_host, bounds_host, loglik, prop, prop_lp,
                                    chains, logpost, n_acc, rows, ld_rows, stream);
}

int elfi_b200_bsl_mh_step_keyed_f64(elfi_b200_ctx* ctx, int64_t C, int64_t p, int64_t t,
                                    int64_t n_samples, int64_t burn_in, int64_t b,
                                    const uint64_t* keys, const uint32_t* lanes,
                                    const double* spec_host, const double* chol_host,
                                    const double* bounds_host, const double* loglik, double* prop,
                                    double* prop_lp, double* chains, double* logpost,
                                    int64_t* n_acc, double* rows, int64_t ld_rows, void* stream) {
    ELFI_REQUIRE(keys && lanes, "bsl_mh_step_keyed: NULL keys or lanes");
    return elfi::bsl_mh_step_launch(ctx, C, p, t, n_samples, burn_in, b, 0, keys, lanes,
                                    spec_host, chol_host, bounds_host, loglik, prop, prop_lp,
                                    chains, logpost, n_acc, rows, ld_rows, stream);
}

}  // extern "C"
