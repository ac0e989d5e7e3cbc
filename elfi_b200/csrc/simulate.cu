// simulate.cu -- device-side generation for the throughput mode (SURVEY.md section 8f, row N2):
// MA2 prior draws, the MA2 simulator fused with its autocovariance summaries, and Gaussian-mixture
// proposals with the MA2 prior support, so that a whole SMC-ABC batch is born in HBM and only
// accepted particles ever leave the device.
//
// Reference functions mirrored (statistically, not bit-wise: the reference draws from a host
// MT19937 RandomState, here a counter-based Philox4x32-10 stream keyed by (seed, batch, row)):
//   elfi/examples/ma2.py:11-37    MA2(t1, t2)              x_i = w_i + t1 w_{i-1} + t2 w_{i-2}
//   elfi/examples/ma2.py:40-59    autocov (lags 1, 2), NumPy pairwise summation order kept
//   elfi/examples/ma2.py:96-186   CustomPrior1 (triangular t1), CustomPrior2 (uniform t2 | t1)
//   elfi/methods/utils.py:200-261 GMDistribution.rvs (choice by weights + MVN perturbation +
//                                 rejection of draws outside the prior support)
// The random numbers are a pure function of (seed, stream, row, index): the simulator can be
// replayed (e.g. to materialise X for a test) and any sharding of rows gives the same particles.
// oracle/streams.py replays every kernel's counter layout in NumPy; tests/test_streams_gpu.py
// compares the kernels with it element by element.

#include "boxmuller.cuh"
#include "gnkmath.cuh"
#include "leafsum.cuh"
#include "pairwise.cuh"
#include "philox.cuh"
#include "priors.cuh"

namespace elfi {

// ---- MA2 prior ------------------------------------------------------------------------------
// mode 0: joint draw (t1, t2); mode 1: t1 only; mode 2: t2 given the t1 passed in.
__global__ void prior_ma2_kernel(int64_t B, uint64_t seed, uint64_t offset, int mode,
                                 double* __restrict__ t1, double* __restrict__ t2) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= B) return;
    const Philox ph(seed);
    const uint64_t row = offset + uint64_t(i);
    const uint4 r = ph(uint32_t(row), uint32_t(row >> 32), 0u, 0x50524931u);
    const double u = u01(r.x, r.y), v = u01(r.z, r.w);
    const double b = 2.0, a = 1.0;
    double x1;
    if (mode == 2) {
        x1 = t1[i];
    } else {
        x1 = u < 0.5 ? sqrt(2.0 * u) * b - b : -sqrt(2.0 * (1.0 - u)) * b + b;
        t1[i] = x1;
    }
    if (mode != 1) {
        const double loc = fmax(-a - x1, -a + x1);
        t2[i] = loc + (a - loc) * v;
    }
}

__device__ __forceinline__ bool ma2_in_support(double x1, double x2) {
    const double ax = fabs(x1);
    return ax < 2.0 && x2 >= -1.0 + ax && x2 <= 1.0;
}

// log p(t1) + log p(t2 | t1) of the MA2 priors (b = 2, a = 1); -inf outside the support
__global__ void logprior_ma2_kernel(const double* __restrict__ x, int64_t ld, int64_t B,
                                    double* __restrict__ out) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= B) return;
    const double x1 = x[i * ld], x2 = x[i * ld + 1];
    const double ax = fabs(x1);
    double lp = -INFINITY;
    if (ma2_in_support(x1, x2)) lp = log(0.5 - ax * 0.25) - log(2.0 - ax);
    out[i] = lp;
}

// Elements k0 + E .. k0 + 7 of a group of eight: their lag-1 / lag-2 products into the leaf sums
// (E is a template parameter because the slot of a product, index % 8, must be static).
template <int E>
__device__ __forceinline__ void ma2_leaf_products(LeafSum& l1, LeafSum& l2, const double (&x)[8],
                                                  double xm1, double xm2, bool mid, int k0,
                                                  int cnt) {
    const double prev1 = (E == 0) ? xm1 : x[E >= 1 ? E - 1 : 0];
    const double prev2 = (E == 0) ? xm2 : (E == 1 ? xm1 : x[E >= 2 ? E - 2 : 0]);
    if (mid) {
        l1.push_mid<(E + 7) & 7>(__dmul_rn(x[E], prev1));
        l2.push_mid<(E + 6) & 7>(__dmul_rn(x[E], prev2));
    } else if (E < cnt) {
        const int k = k0 + E;
        if (k >= 1) l1.push<(E + 7) & 7>(k - 1, __dmul_rn(x[E], prev1));
        if (k >= 2) l2.push<(E + 6) & 7>(k - 2, __dmul_rn(x[E], prev2));
    }
    if constexpr (E + 1 < 8) ma2_leaf_products<E + 1>(l1, l2, x, xm1, xm2, mid, k0, cnt);
}

// ---- MA2 simulator (+ fused autocovariance) ---------------------------------------------------
// One thread per row; normals are generated eight at a time (4 Philox blocks).
// LEAF: both product rows fit one leaf of NumPy's pairwise sum (n_obs - 1 <= 128, e.g. the 99 / 98
// products of the benchmark model): eight running sums per lag (leafsum.cuh) instead of the general
// PairwiseStream tree with its per-level stack -- the kernel drops from 255 registers to well under
// half, i.e. more than two resident blocks per SM for a kernel whose Box-Muller chains need the
// latency hiding (the kernel is latency bound, not fp64-pipe bound).
template <bool WRITE_X, bool SUMMARIES, bool LEAF>
__global__ void __launch_bounds__(128)
sim_ma2_kernel(const double* __restrict__ t1, const double* __restrict__ t2, int64_t B, int n_obs,
               uint64_t seed, uint64_t offset, double* __restrict__ X, int64_t ldX,
               double* __restrict__ S, int64_t ldS) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= B) return;
    const Philox ph(seed);
    const uint64_t row = offset + uint64_t(i);
    const uint32_t r0 = uint32_t(row), r1 = uint32_t(row >> 32);
    const double a1 = t1[i], a2 = t2[i];
    PairwiseStream<6> p1, p2;      // lag-1 and lag-2 product sums (rows up to 7688 terms)
    LeafSum l1, l2;                // the same sums when a row is a single leaf
    if (SUMMARIES) {
        if constexpr (LEAF) {
            l1.begin(n_obs - 1);
            l2.begin(n_obs - 2);
        } else {
            p1.begin(n_obs - 1);
            p2.begin(n_obs - 2);
        }
    }
    // w has n_obs + 2 entries; x_k = w_{k+2} + a1 w_{k+1} + a2 w_k
    double wm2, wm1;   // w_{k}, w_{k+1} before the current group
    {
        double n0, n1;
        normal2(ph(r0, r1, 0u, 0x4d413257u), n0, n1);
        wm2 = n0;
        wm1 = n1;
    }
    double xm1 = 0.0, xm2 = 0.0;   // x_{k-1}, x_{k-2}
    double b1[8], b2[8];
    for (int k0 = 0; k0 < n_obs; k0 += 8) {
        double w[8];
#pragma unroll
        for (int q = 0; q < 4; ++q)
            normal2(ph(r0, r1, uint32_t(1 + (k0 >> 1) + q), 0x4d413257u), w[2 * q], w[2 * q + 1]);
        double x[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const double wk = (e == 0) ? wm2 : (e == 1 ? wm1 : w[e >= 2 ? e - 2 : 0]);
            const double wk1 = (e == 0) ? wm1 : w[e >= 1 ? e - 1 : 0];
            // (w2 + t1*w1) + t2*w0 with separate roundings, like the NumPy expression in ma2.py:36
            x[e] = __dadd_rn(__dadd_rn(w[e], __dmul_rn(a1, wk1)), __dmul_rn(a2, wk));
        }
        wm2 = w[6];
        wm1 = w[7];
        const int cnt = (n_obs - k0) < 8 ? (n_obs - k0) : 8;
        if (WRITE_X) {
#pragma unroll
            for (int e = 0; e < 8; ++e)
                if (e < cnt) X[i * ldX + k0 + e] = x[e];
        }
        if constexpr (SUMMARIES && LEAF) {
            // product index k - 1 (lag 1) / k - 2 (lag 2) of element k = k0 + e goes straight into
            // its running sum; slot = index % 8 is static because k0 is a multiple of 8
            const bool mid = cnt == 8 && l1.all_mid(k0 - 1, k0 + 6) && l2.all_mid(k0 - 2, k0 + 5);
            ma2_leaf_products<0>(l1, l2, x, xm1, xm2, mid, k0, cnt);
        }
        if constexpr (SUMMARIES && !LEAF) {
            // lag-1 products p[j] = x[j+1] x[j], j = k - 1 for element k; lag-2: j = k - 2.
            // Feed aligned groups of 8 products: group g of lag 1 needs x[8g .. 8g+8].
            // b1[] holds products with indices 8(g) .. 8g+7 once x[8g+8] is known, so products are
            // emitted one group late: element k contributes product index k-1 (lag 1), k-2 (lag 2).
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const int k = k0 + e;
                if (e < cnt) {
                    const double prev1 = (e == 0) ? xm1 : x[e >= 1 ? e - 1 : 0];
                    const double prev2 = (e == 0) ? xm2 : (e == 1 ? xm1 : x[e >= 2 ? e - 2 : 0]);
                    // product index for lag 1 is k-1: slot (k-1) & 7 == (e + 7) & 7
                    if (k >= 1) {
                        b1[(e + 7) & 7] = __dmul_rn(x[e], prev1);
                        if (((e + 7) & 7) == 7) p1.feed8(k - 8, b1, 8);
                    }
                    if (k >= 2) {
                        b2[(e + 6) & 7] = __dmul_rn(x[e], prev2);
                        if (((e + 6) & 7) == 7) p2.feed8(k - 9, b2, 8);
                    }
                }
            }
        }
        xm2 = x[6];
        xm1 = x[7];
    }
    if constexpr (SUMMARIES && LEAF) {
        S[i * ldS + 0] = l1.finish(n_obs - 1) / double(n_obs - 1);
        S[i * ldS + 1] = l2.finish(n_obs - 2) / double(n_obs - 2);
    }
    if constexpr (SUMMARIES && !LEAF) {
        const int m1 = n_obs - 1, m2 = n_obs - 2;
        if (m1 % 8) p1.feed8(m1 - m1 % 8, b1, m1 % 8);
        if (m2 % 8) p2.feed8(m2 - m2 % 8, b2, m2 % 8);
        S[i * ldS + 0] = p1.finish() / double(m1);
        S[i * ldS + 1] = p2.finish() / double(m2);
    }
}

// ---- Gaussian-mixture proposals ------------------------------------------------------------------
// cumw: inclusive cumulative sum of the normalised weights (N); Lc: lower Cholesky factor of the
// shared covariance (p x p, row-major, p <= 4).  support: 0 none, 1 MA2 prior support, 2 box.
// Support 3 and p > 4 go to gm_rvs_wide_kernel below; this kernel is the p <= 4 path as it was.
struct BoxSupport { double lo[4], hi[4]; };
struct LowerFactor4 { double v[16]; };   // row-major p x p (p <= 4), passed by value

__global__ void gm_rvs_kernel(const double* __restrict__ means, int64_t ldm, const double* __restrict__ cumw,
                              int64_t N, int p, const LowerFactor4 Lc, int64_t B,
                              uint64_t seed, uint64_t offset, int support, BoxSupport box,
                              double* __restrict__ out, int64_t ldo) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= B) return;
    const Philox ph(seed);
    const uint64_t row = offset + uint64_t(i);
    const double total = cumw[N - 1];
    double x[4];
    for (uint32_t trial = 0; trial < 1000u; ++trial) {
        const uint4 r = ph(uint32_t(row), uint32_t(row >> 32), trial * 4u, 0x474d5256u);
        const double u = u01(r.x, r.y) * total;
        int64_t lo = 0, hi = N - 1;               // first index with cumw >= u
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (cumw[mid] < u) lo = mid + 1; else hi = mid;
        }
        double z[4];
        normal2(ph(uint32_t(row), uint32_t(row >> 32), trial * 4u + 1u, 0x474d5256u), z[0], z[1]);
        if (p > 2) normal2(ph(uint32_t(row), uint32_t(row >> 32), trial * 4u + 2u, 0x474d5256u), z[2], z[3]);
        for (int a = 0; a < p; ++a) {
            double s = means[lo * ldm + a];
            for (int b = 0; b <= a; ++b) s = fma(Lc.v[a * p + b], z[b], s);
            x[a] = s;
        }
        bool ok = support == 0 || (support == 1 && ma2_in_support(x[0], x[1]));
        if (support == 2) {
            ok = true;
            for (int a = 0; a < p; ++a) ok = ok && x[a] >= box.lo[a] && x[a] <= box.hi[a];
        }
        if (ok) break;
    }
    for (int a = 0; a < p; ++a) out[i * ldo + a] = x[a];
}

// The same proposals for p <= 16 and for support 3, "prior": a draw is kept iff the joint log
// density of the prior table (priors.cuh) is finite, the rule of GMDistribution.rvs
// (x[np.isfinite(prior_logpdf(x))], utils.py:200-261); a conditional entry's loc / scale is
// read from the draw's own columns (support 4 on the host side).  Trial t uses blocks 4t .. 4t + 2 of
// SALT_GM_RVS exactly as gm_rvs_kernel does (component uniform, z_0 z_1, z_2 z_3), so for p <= 4
// the two kernels draw the same particles; z_{4+2k}, z_{5+2k} come from block 8t + k of
// SALT_GM_RVS_WIDE (k = 0 .. 5).  The factor is packed: row a of L starts at a (a + 1) / 2.
constexpr uint32_t SALT_GM_RVS = 0x474d5256u, SALT_GM_RVS_WIDE = 0x474d5258u;
struct PackedLower16 { double v[PRIOR_MAX_PARAMS * (PRIOR_MAX_PARAMS + 1) / 2]; };
struct BoxSupport16 { double lo[PRIOR_MAX_PARAMS], hi[PRIOR_MAX_PARAMS]; };

// PMAX (4, 8 or 16) >= p: the loops are unrolled over PMAX so that x[] and z[] stay in registers.
// COND: the prior table has conditional entries (support 4); without them the sources are
// compiled out (at PMAX 16 resolving them takes 168 registers instead of 96).
template <int PMAX, bool COND>
__global__ void __launch_bounds__(128)
gm_rvs_wide_kernel(const double* __restrict__ means, int64_t ldm, const double* __restrict__ cumw,
                   int64_t N, int p, const PackedLower16 Lc, int64_t B, uint64_t seed,
                   uint64_t offset, int support, const BoxSupport16 box, const PriorTable prior,
                   double* __restrict__ out, int64_t ldo) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= B) return;
    const Philox ph(seed);
    const uint64_t row = offset + uint64_t(i);
    const uint32_t r0 = uint32_t(row), r1 = uint32_t(row >> 32);
    const double total = cumw[N - 1];
    double x[PMAX];
    for (uint32_t trial = 0; trial < 1000u; ++trial) {
        const uint4 r = ph(r0, r1, trial * 4u, SALT_GM_RVS);
        const double u = u01(r.x, r.y) * total;
        int64_t lo = 0, hi = N - 1;               // first index with cumw >= u
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (cumw[mid] < u) lo = mid + 1; else hi = mid;
        }
        double z[PMAX];
        normal2(ph(r0, r1, trial * 4u + 1u, SALT_GM_RVS), z[0], z[1]);
        if (p > 2) normal2(ph(r0, r1, trial * 4u + 2u, SALT_GM_RVS), z[2], z[3]);
#pragma unroll
        for (int k = 0; k < (PMAX - 4) / 2; ++k)
            if (4 + 2 * k < p) normal2(ph(r0, r1, trial * 8u + uint32_t(k), SALT_GM_RVS_WIDE),
                                       z[4 + 2 * k], z[5 + 2 * k]);
#pragma unroll
        for (int a = 0; a < PMAX; ++a) {
            if (a < p) {
                double s = means[lo * ldm + a];
#pragma unroll
                for (int b = 0; b <= a; ++b) s = fma(Lc.v[a * (a + 1) / 2 + b], z[b], s);
                x[a] = s;
            }
        }
        bool ok = true;
        if (support == 2) {
#pragma unroll
            for (int a = 0; a < PMAX; ++a)
                if (a < p) ok = ok && x[a] >= box.lo[a] && x[a] <= box.hi[a];
        } else if (support == 3) {
            ok = isfinite(prior_joint_logpdf<PMAX, COND>(prior.e, x, p));
        }
        if (ok) break;
    }
#pragma unroll
    for (int a = 0; a < PMAX; ++a)
        if (a < p) out[i * ldo + a] = x[a];
}

// ---- Gaussian noise model (elfi/examples/gauss.py) --------------------------------------------------
// priors of get_model(): mu ~ U(mu_lo, mu_lo + mu_w); sigma ~ truncnorm(a, b) (standard normal
// truncated to [a, b], scipy convention with loc 0, scale 1).  sigma is drawn by inverse-CDF
// sampling of [lo, hi] = [a, b] with the result multiplied by sign = 1 or, when a > 0, of the
// mirror image [-b, -a] with sign = -1: in the upper tail Phi(a) rounds to 1 (a >~ 8.3) and
// Phi(b) - Phi(a) loses every digit, while Phi(-a) and Phi(-b) stay accurate.
// cdf_lo = Phi(lo), cdf_w = Phi(hi) - Phi(lo) (the mass of the truncation).
struct GaussPrior { double mu_lo, mu_w, a, b, lo, hi, sign, cdf_lo, cdf_w; };

__global__ void prior_gauss_kernel(int64_t B, uint64_t seed, uint64_t offset, GaussPrior g,
                                   double* __restrict__ mu, double* __restrict__ sigma) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= B) return;
    const Philox ph(seed);
    const uint64_t row = offset + uint64_t(i);
    const uint4 r = ph(uint32_t(row), uint32_t(row >> 32), 0u, 0x47415553u);
    const double u = u01(r.x, r.y), v = u01(r.z, r.w);
    mu[i] = g.mu_lo + g.mu_w * u;
    double sgm = normcdfinv(g.cdf_lo + v * g.cdf_w);    // inverse-CDF sampling of the truncation
    sigma[i] = g.sign * fmin(fmax(sgm, g.lo), g.hi);
}

__global__ void logprior_gauss_kernel(const double* __restrict__ x, int64_t ld, int64_t B, GaussPrior g,
                                      double* __restrict__ out) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= B) return;
    const double m = x[i * ld], s = x[i * ld + 1];
    double lp = -INFINITY;
    if (m >= g.mu_lo && m <= g.mu_lo + g.mu_w && s >= g.a && s <= g.b)
        lp = -log(g.mu_w) - 0.5 * s * s - 0.9189385332046727 - log(g.cdf_w);
    out[i] = lp;
}

// y_ij = mu_i + sigma_i z_ij (gauss.py:11-35) with np.mean / np.var summaries (gauss.py:142-173,
// NumPy pairwise order).  The variance needs the mean first: the counter-based normals are simply
// generated a second time instead of being stored.
// Terms k0 + E .. k0 + 7 of a group of eight into a single-leaf sum (static slots).
template <int E>
__device__ __forceinline__ void leaf_feed8(LeafSum& s, int k0, const double (&t)[8], int cnt,
                                           bool mid) {
    if (mid) s.push_mid<E>(t[E]);
    else if (E < cnt) s.push<E>(k0 + E, t[E]);
    if constexpr (E + 1 < 8) leaf_feed8<E + 1>(s, k0, t, cnt, mid);
}

// LEAF: n_obs <= 128, the row sums are single leaves of NumPy's pairwise sum (fewer registers, more
// resident blocks; keeping the draws in registers to generate them only once was tried and is
// slower -- 180 registers, two blocks per SM: the Box-Muller chains need the occupancy more than
// they need the halved work).
template <bool WRITE_Y, bool LEAF>
__global__ void __launch_bounds__(128)
sim_gauss_kernel(const double* __restrict__ mu, const double* __restrict__ sigma, int64_t B, int n_obs,
                 uint64_t seed, uint64_t offset, double* __restrict__ Y, int64_t ldY,
                 double* __restrict__ S, int64_t ldS) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= B) return;
    const Philox ph(seed);
    const uint64_t row = offset + uint64_t(i);
    const uint32_t r0 = uint32_t(row), r1 = uint32_t(row >> 32);
    const double m = mu[i], sg = sigma[i];
    PairwiseStream<6> pw;
    LeafSum lf;
    double mean = 0.0;
    for (int pass = 0; pass < (S ? 2 : 1); ++pass) {
        if (S) {
            if constexpr (LEAF) lf.begin(n_obs); else pw.begin(n_obs);
        }
        double t[8];
        for (int k0 = 0; k0 < n_obs; k0 += 8) {
            double y[8];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                double z0, z1;
                normal2(ph(r0, r1, uint32_t((k0 >> 1) + q), 0x47534d55u), z0, z1);
                y[2 * q] = __dadd_rn(m, __dmul_rn(sg, z0));
                y[2 * q + 1] = __dadd_rn(m, __dmul_rn(sg, z1));
            }
            const int cnt = (n_obs - k0) < 8 ? (n_obs - k0) : 8;
            if (WRITE_Y && pass == 0) {
#pragma unroll
                for (int e = 0; e < 8; ++e)
                    if (e < cnt) Y[i * ldY + k0 + e] = y[e];
            }
            if (S) {
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    if (pass == 0) {
                        t[e] = y[e];
                    } else {
                        const double c = __dsub_rn(y[e], mean);
                        t[e] = __dmul_rn(c, c);
                    }
                }
                if constexpr (LEAF)
                    leaf_feed8<0>(lf, k0, t, cnt, cnt == 8 && lf.all_mid(k0, k0 + 7));
                else
                    pw.feed8(k0, t, cnt);
            }
        }
        if (S) {
            const double v = (LEAF ? lf.finish(n_obs) : pw.finish()) / double(n_obs);
            if (pass == 0) { mean = v; S[i * ldS] = v; } else { S[i * ldS + 1] = v; }
        }
    }
}

// ---- g-and-k model (elfi/examples/gnk.py) -------------------------------------------------------
// y_ij = Q(z_ij; A_i, B_i, g_i, k_i, c) with the quantile function of gnkmath.cuh (gnk.py:60-66).
// One thread per pair of observations: Philox block (row, pair) -> two normals -> two adjacent
// outputs, so a warp writes 512 contiguous bytes of a row.  The draws of a row do not depend on
// n_obs or on how rows are sharded.
__global__ void __launch_bounds__(256)
sim_gnk_kernel(const double* __restrict__ A, const double* __restrict__ Bs, const double* __restrict__ g,
               const double* __restrict__ k, double c, int64_t B, int n_obs, uint64_t seed,
               uint64_t offset, double* __restrict__ Y, int64_t ldY) {
    const int half = (n_obs + 1) >> 1;
    const int64_t total = B * half;
    const Philox ph(seed);
    const bool vec = (ldY & 1) == 0 && (reinterpret_cast<uintptr_t>(Y) & 15) == 0;
    for (int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
         idx += int64_t(gridDim.x) * blockDim.x) {
        const int64_t i = idx / half;
        const int q = int(idx - i * half);
        const uint64_t row = offset + uint64_t(i);
        double z0, z1;
        normal2(ph(uint32_t(row), uint32_t(row >> 32), uint32_t(q), 0x474e4b30u), z0, z1);
        const double a = A[i], b = Bs[i], gg = g[i], kk = k[i];
        const double y0 = gnk_quantile(a, b, gg, kk, c, z0);
        double* dst = Y + i * ldY + 2 * q;
        if (2 * q + 1 < n_obs) {
            const double y1 = gnk_quantile(a, b, gg, kk, c, z1);
            if (vec) {
                *reinterpret_cast<double2*>(dst) = make_double2(y0, y1);
            } else {
                dst[0] = y0;
                dst[1] = y1;
            }
        } else {
            dst[0] = y0;
        }
    }
}

// log density of independent uniform priors U(lo_a, lo_a + width_a), a < p <= 8
// (gnk.py:99-103: A, B, g, k ~ uniform(0, 10)); -inf outside the box like scipy's logpdf.
struct BoxPrior { double lo[8], hi[8]; double logdens; };

__global__ void logprior_box_kernel(const double* __restrict__ x, int64_t ld, int64_t B, int p,
                                    BoxPrior box, double* __restrict__ out) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= B) return;
    bool inside = true;
    for (int a = 0; a < p; ++a) {
        const double v = x[i * ld + a];
        inside = inside && v >= box.lo[a] && v <= box.hi[a];   // NaN -> outside
    }
    out[i] = inside ? box.logdens : -INFINITY;
}

// Inclusive running sum of the (unnormalised) weights, w == NULL: all ones; single block, N up to
// a few million.  A tile is 1024 threads x GM_CDF_PER_THREAD consecutive weights: each thread adds
// its weights sequentially, the thread totals are scanned (warp shuffles, then the warp totals left
// to right) into each thread's base, and the running sums from that base are capped below by a
// running maximum of the threads' last values.  The table is therefore nondecreasing, which the
// binary search of gm_rvs_kernel needs: a plain tree scan adds in a different order for
// neighbouring entries, and after a zero weight an entry can round one ulp below its predecessor,
// so that the search skips the right component or lands on a zero-weight one.  Only additions in
// a fixed order and maxima: the table is a deterministic function of the weights
// (oracle/streams.py gm_cdf replays it bit for bit).
constexpr int GM_CDF_PER_THREAD = 8;

__global__ void __launch_bounds__(1024)
cumsum_kernel(const double* __restrict__ w, int64_t n, double* __restrict__ out) {
    constexpr int K = GM_CDF_PER_THREAD;
    __shared__ double wsum[32], wmax[32];
    __shared__ double carry_s;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) carry_s = 0.0;
    __syncthreads();
    for (int64_t base = 0; base < n; base += 1024 * K) {
        const int64_t i0 = base + int64_t(tid) * K;
        double v[K];
#pragma unroll
        for (int j = 0; j < K; ++j) v[j] = i0 + j < n ? (w ? w[i0 + j] : 1.0) : 0.0;
        double tot = v[0];
#pragma unroll
        for (int j = 1; j < K; ++j) tot += v[j];
        double incl = tot;
        for (int o = 1; o < 32; o <<= 1) {
            const double t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        double excl = __shfl_up_sync(0xffffffffu, incl, 1);
        if (lane == 0) excl = 0.0;
        if (lane == 31) wsum[wid] = incl;
        __syncthreads();
        double woff = 0.0;
        for (int k = 0; k < wid; ++k) woff += wsum[k];
        const double carry = carry_s;
        double run = carry + (woff + excl);
        double r[K];
        bool seen = false;                     // a nonzero weight among this thread's so far
#pragma unroll
        for (int j = 0; j < K; ++j) {
            run += v[j];
            seen = seen || v[j] != 0.0;
            r[j] = seen ? run : -INFINITY;
        }
        // exclusive running maximum of the threads' last values, starting at the carry.  A
        // thread's leading zero weights take that maximum, which is exactly the entry before
        // them: a zero weight never gets a share of the table, not even one ulp.
        double m = r[K - 1];
        for (int o = 1; o < 32; o <<= 1) {
            const double t = __shfl_up_sync(0xffffffffu, m, o);
            if (lane >= o) m = fmax(m, t);
        }
        double pm = __shfl_up_sync(0xffffffffu, m, 1);
        if (lane == 0) pm = carry;
        if (lane == 31) wmax[wid] = m;
        __syncthreads();
        pm = fmax(pm, carry);
        for (int k = 0; k < wid; ++k) pm = fmax(pm, wmax[k]);
#pragma unroll
        for (int j = 0; j < K; ++j)
            if (i0 + j < n) out[i0 + j] = fmax(r[j], pm);
        __syncthreads();                       // carry_s, wsum and wmax have been read
        if (tid == 1023) carry_s = fmax(r[K - 1], pm);
        __syncthreads();
    }
}

}  // namespace elfi

extern "C" {

int elfi_b200_prior_ma2_f64(elfi_b200_ctx* ctx, int64_t B, uint64_t seed, uint64_t offset,
                            int32_t mode, double* t1, double* t2, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && mode >= 0 && mode <= 2, "prior_ma2: bad argument");
    ELFI_REQUIRE(B == 0 || (t1 && (mode == 1 || t2)), "prior_ma2: NULL argument");
    if (B == 0) return ELFI_B200_OK;
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        prior_ma2_kernel<<<unsigned((B + 255) / 256), 256, 0, stream>>>(B, seed, offset, mode, t1,
                                                                        t2);
        return ELFI_B200_OK;
    });
}

int elfi_b200_logprior_ma2_f64(elfi_b200_ctx* ctx, const double* x, int64_t ldx, int64_t B,
                               double* out, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || (x && out)) && ldx >= 2, "logprior_ma2: bad argument");
    if (B == 0) return ELFI_B200_OK;
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        logprior_ma2_kernel<<<unsigned((B + 255) / 256), 256, 0, stream>>>(x, ldx, B, out);
        return ELFI_B200_OK;
    });
}

int elfi_b200_sim_ma2_f64(elfi_b200_ctx* ctx, const double* t1, const double* t2, int64_t B,
                          int64_t n_obs, uint64_t seed, uint64_t offset, double* X, int64_t ldX,
                          double* S, int64_t ldS, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || (t1 && t2)), "sim_ma2: NULL argument");
    ELFI_REQUIRE(n_obs >= 3 && n_obs <= PairwiseStream<6>::max_terms(),
                 "sim_ma2: n_obs=%lld outside [3, 7688]", (long long)n_obs);
    ELFI_REQUIRE(X || S, "sim_ma2: nothing to produce (X and S are both NULL)");
    ELFI_REQUIRE((!X || ldX >= n_obs) && (!S || ldS >= 2), "sim_ma2: bad leading dimension");
    if (B == 0) return ELFI_B200_OK;
    const unsigned blocks = unsigned((B + 127) / 128);
    const bool leaf = n_obs - 1 <= LEAF_MAX_TERMS;
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
#define ELFI_SIM_MA2(WX, SM, LF) \
    sim_ma2_kernel<WX, SM, LF><<<blocks, 128, 0, stream>>>(t1, t2, B, int(n_obs), seed, offset, X, ldX, S, ldS)
        if (X && S) { if (leaf) ELFI_SIM_MA2(true, true, true); else ELFI_SIM_MA2(true, true, false); }
        else if (X) ELFI_SIM_MA2(true, false, false);
        else { if (leaf) ELFI_SIM_MA2(false, true, true); else ELFI_SIM_MA2(false, true, false); }
#undef ELFI_SIM_MA2
        return ELFI_B200_OK;
    });
}

int elfi_b200_gm_cdf_f64(elfi_b200_ctx* ctx, const double* weights, int64_t N, double* cumw,
                         void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && cumw && N >= 1, "gm_cdf: bad argument");
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        cumsum_kernel<<<1, 1024, 0, stream>>>(weights, N, cumw);
        return ELFI_B200_OK;
    });
}

int elfi_b200_gm_rvs_cdf_f64(elfi_b200_ctx* ctx, const double* means, int64_t ldm, const double* cumw,
                             int64_t N, int64_t p, const double* Lchol_host, int64_t B, uint64_t seed,
                             uint64_t offset, int32_t support, const double* box_host, double* out,
                             int64_t ldo, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && means && cumw && Lchol_host && (B == 0 || out), "gm_rvs: NULL argument");
    ELFI_REQUIRE(N >= 1 && p >= 1 && p <= PRIOR_MAX_PARAMS && ldm >= p && ldo >= p,
                 "gm_rvs: bad shape (p <= 16)");
    ELFI_REQUIRE(support == 0 || (support == 1 && p == 2) ||
                     ((support == 2 || support == 3 || support == 4) && box_host),
                 "gm_rvs: unknown support %d", support);
    if (support >= 3 || p > 4) {
        // the wide kernel: support 3 or 4 (the prior table of 5 or 7 words per parameter travels
        // in box_host; the kernel treats both as support 3) or p > 4
        PriorTable prior;
        memset(&prior, 0, sizeof(prior));
        const bool cond = support == 4;
        if (support >= 3) {
            for (int a = 0; a < p; ++a) {
                char why[200];
                const bool ok =
                    support == 4
                        ? prior_entry_from_spec7(box_host + PRIOR_COND_SPEC_WORDS * a, a, int(p),
                                                 &prior.e[a], why, sizeof(why))
                        : prior_entry_from_spec(box_host + PRIOR_SPEC_WORDS * a, &prior.e[a], why,
                                                sizeof(why));
                ELFI_REQUIRE(ok, "gm_rvs: prior parameter %d: %s", a, why);
            }
            support = 3;
        }
        BoxSupport16 box16;
        memset(&box16, 0, sizeof(box16));
        if (support == 2)
            for (int a = 0; a < p; ++a) { box16.lo[a] = box_host[a]; box16.hi[a] = box_host[p + a]; }
        if (B == 0) return ELFI_B200_OK;
        PackedLower16 Lp;
        memset(&Lp, 0, sizeof(Lp));
        for (int a = 0; a < p; ++a)
            for (int b = 0; b <= a; ++b) Lp.v[a * (a + 1) / 2 + b] = Lchol_host[a * p + b];
        return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
#define ELFI_GM_RVS_WIDE(PMAX, COND)                                                             \
            gm_rvs_wide_kernel<PMAX, COND><<<unsigned((B + 127) / 128), 128, 0, stream>>>(        \
                means, ldm, cumw, N, int(p), Lp, B, seed, offset, support, box16, prior, out, ldo)
            if (p <= 4) { if (cond) ELFI_GM_RVS_WIDE(4, true); else ELFI_GM_RVS_WIDE(4, false); }
            else if (p <= 8) { if (cond) ELFI_GM_RVS_WIDE(8, true); else ELFI_GM_RVS_WIDE(8, false); }
            else if (cond) ELFI_GM_RVS_WIDE(16, true);
            else ELFI_GM_RVS_WIDE(16, false);
#undef ELFI_GM_RVS_WIDE
            return ELFI_B200_OK;
        });
    }
    BoxSupport box;
    memset(&box, 0, sizeof(box));
    if (support == 2)
        for (int a = 0; a < p; ++a) { box.lo[a] = box_host[a]; box.hi[a] = box_host[p + a]; }
    if (B == 0) return ELFI_B200_OK;
    LowerFactor4 Lc;
    memset(&Lc, 0, sizeof(Lc));
    for (int a = 0; a < p; ++a)
        for (int b = 0; b <= a; ++b) Lc.v[a * p + b] = Lchol_host[a * p + b];
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        gm_rvs_kernel<<<unsigned((B + 127) / 128), 128, 0, stream>>>(
            means, ldm, cumw, N, int(p), Lc, B, seed, offset, support, box, out, ldo);
        return ELFI_B200_OK;
    });
}

static elfi::GaussPrior make_gauss_prior(const double* prm) {
    elfi::GaussPrior g;
    g.mu_lo = prm[0]; g.mu_w = prm[1]; g.a = prm[2]; g.b = prm[3];
    const bool mirror = g.a > 0.0;
    g.lo = mirror ? -g.b : g.a;
    g.hi = mirror ? -g.a : g.b;
    g.sign = mirror ? -1.0 : 1.0;
    g.cdf_lo = 0.5 * erfc(-g.lo * 0.7071067811865476);
    g.cdf_w = 0.5 * erfc(-g.hi * 0.7071067811865476) - g.cdf_lo;
    return g;
}

/* prm_host = [mu_lo, mu_width, a, b] of mu ~ U(mu_lo, mu_lo + mu_width), sigma ~ truncnorm(a, b) */
int elfi_b200_prior_gauss_f64(elfi_b200_ctx* ctx, int64_t B, uint64_t seed, uint64_t offset,
                              const double* prm_host, double* mu, double* sigma, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && prm_host && (B == 0 || (mu && sigma)), "prior_gauss: NULL argument");
    ELFI_REQUIRE(prm_host[1] > 0 && prm_host[3] > prm_host[2], "prior_gauss: bad prior parameters");
    if (B == 0) return ELFI_B200_OK;
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        prior_gauss_kernel<<<unsigned((B + 255) / 256), 256, 0, stream>>>(
            B, seed, offset, make_gauss_prior(prm_host), mu, sigma);
        return ELFI_B200_OK;
    });
}

int elfi_b200_logprior_gauss_f64(elfi_b200_ctx* ctx, const double* x, int64_t ldx, int64_t B,
                                 const double* prm_host, double* out, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && prm_host && (B == 0 || (x && out)) && ldx >= 2, "logprior_gauss: bad argument");
    if (B == 0) return ELFI_B200_OK;
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        logprior_gauss_kernel<<<unsigned((B + 255) / 256), 256, 0, stream>>>(
            x, ldx, B, make_gauss_prior(prm_host), out);
        return ELFI_B200_OK;
    });
}

int elfi_b200_sim_gauss_f64(elfi_b200_ctx* ctx, const double* mu, const double* sigma, int64_t B,
                            int64_t n_obs, uint64_t seed, uint64_t offset, double* Y, int64_t ldY,
                            double* S, int64_t ldS, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || (mu && sigma)), "sim_gauss: NULL argument");
    ELFI_REQUIRE(n_obs >= 1 && n_obs <= PairwiseStream<6>::max_terms(),
                 "sim_gauss: n_obs=%lld outside [1, 7688]", (long long)n_obs);
    ELFI_REQUIRE(Y || S, "sim_gauss: nothing to produce (Y and S are both NULL)");
    ELFI_REQUIRE((!Y || ldY >= n_obs) && (!S || ldS >= 2), "sim_gauss: bad leading dimension");
    if (B == 0) return ELFI_B200_OK;
    const unsigned blocks = unsigned((B + 127) / 128);
    const bool leaf = n_obs <= LEAF_MAX_TERMS;
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
#define ELFI_SIM_GAUSS(WY, LF) \
    sim_gauss_kernel<WY, LF><<<blocks, 128, 0, stream>>>(mu, sigma, B, int(n_obs), seed, offset, Y, ldY, S, ldS)
        if (Y) { if (leaf) ELFI_SIM_GAUSS(true, true); else ELFI_SIM_GAUSS(true, false); }
        else { if (leaf) ELFI_SIM_GAUSS(false, true); else ELFI_SIM_GAUSS(false, false); }
#undef ELFI_SIM_GAUSS
        return ELFI_B200_OK;
    });
}

int elfi_b200_sim_gnk_f64(elfi_b200_ctx* ctx, const double* A, const double* Bs, const double* g,
                          const double* k, double c, int64_t B, int64_t n_obs, uint64_t seed,
                          uint64_t offset, double* Y, int64_t ldY, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && (B == 0 || (A && Bs && g && k && Y)), "sim_gnk: NULL argument");
    ELFI_REQUIRE(B >= 0 && n_obs >= 1 && n_obs < (int64_t(1) << 30), "sim_gnk: bad shape B=%lld n_obs=%lld",
                 (long long)B, (long long)n_obs);
    ELFI_REQUIRE(ldY >= n_obs, "sim_gnk: bad leading dimension");
    if (B == 0) return ELFI_B200_OK;
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        // grid-stride beyond 8 waves of 8 CTAs/SM
        const unsigned blocks = capped_grid(ctx, B * ((n_obs + 1) / 2), 256, 64);
        sim_gnk_kernel<<<blocks, 256, 0, stream>>>(A, Bs, g, k, c, B, int(n_obs), seed, offset, Y,
                                                   ldY);
        return ELFI_B200_OK;
    });
}

int elfi_b200_logprior_box_f64(elfi_b200_ctx* ctx, const double* x, int64_t ldx, int64_t B, int64_t p,
                               const double* box_host, double* out, void* stream_) {
    using namespace elfi;
    ELFI_REQUIRE(ctx && box_host && (B == 0 || (x && out)), "logprior_box: NULL argument");
    ELFI_REQUIRE(B >= 0 && p >= 1 && p <= 8 && ldx >= p, "logprior_box: bad shape (p <= 8)");
    BoxPrior box;
    memset(&box, 0, sizeof(box));
    box.logdens = 0.0;
    for (int a = 0; a < p; ++a) {
        ELFI_REQUIRE(box_host[p + a] > 0.0, "logprior_box: width[%d] must be positive", a);
        box.lo[a] = box_host[a];
        box.hi[a] = box_host[a] + box_host[p + a];
        box.logdens -= log(box_host[p + a]);
    }
    if (B == 0) return ELFI_B200_OK;
    return run_on_device(ctx, stream_, [&](cudaStream_t stream) {
        logprior_box_kernel<<<unsigned((B + 255) / 256), 256, 0, stream>>>(x, ldx, B, int(p), box,
                                                                           out);
        return ELFI_B200_OK;
    });
}

}  // extern "C"
