/*
 * elfi_oracle.c -- CPU restatement of the arithmetic on ELFI's sampler hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs may load this library; the product
 * (elfi_b200/) never does and has no CPU fallback.
 *
 * Every function names the reference call site it restates (paths relative to
 * elfi-dev/elfi).  The arithmetic that lives in third-party code (SciPy cdist,
 * NumPy pairwise reductions) is restated from the published algorithm and pinned
 * bit-for-bit against the installed scipy 1.18.1 / numpy 2.3.5 by
 * tests/test_oracle.py (those packages are what the reference itself calls).
 *
 * Build:  gcc -O2 -fPIC -shared -ffp-contract=off   (see oracle/Makefile; threads come from the
 *         Python side: ctypes drops the GIL, callers split rows across a thread pool)
 * -ffp-contract=off matters: the reference's wheels are built for baseline x86-64
 * (no FMA contraction), so every multiply and add below rounds separately.
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* --------------------------------------------------------------------------
 * scipy.spatial.distance.cdist(XA, XB, 'euclidean'[, w=w]) with XB of one row.
 * Call sites: elfi/model/elfi_model.py:1037 (Distance), :1084 and :1131
 * (AdaptiveDistance, w = 1/scale**2), reached through
 * elfi/model/utils.py:37-52 (distance_as_discrepancy).
 * SciPy's kernel walks each row strictly left to right in double precision:
 *   unweighted: acc += (x-o)*(x-o)        weighted: acc += w*((x-o)*(x-o))
 * then sqrt(acc).  No pairwise / SIMD reassociation across a row.
 * ------------------------------------------------------------------------ */
void oracle_cdist_euclid(const double *S, int64_t ld, int64_t B, int64_t D,
                         const double *obs, const double *w, double *out)
{
    for (int64_t i = 0; i < B; ++i) {
        const double *row = S + i * ld;
        double acc = 0.0;
        if (w) {
            for (int64_t j = 0; j < D; ++j) {
                double diff = fabs(row[j] - obs[j]);
                acc += w[j] * (diff * diff);
            }
        } else {
            for (int64_t j = 0; j < D; ++j) {
                double diff = fabs(row[j] - obs[j]);
                acc += diff * diff;
            }
        }
        out[i] = sqrt(acc);
    }
}

/* K nested distance columns (elfi/model/elfi_model.py:1135-1151, nested_distance):
 * column k uses weight row W[k] (W[k][0] is NaN-tagged "None" => unweighted).
 * `unweighted[k]` != 0 selects the unweighted form for column k. out is (B, K). */
void oracle_nested_distance(const double *S, int64_t ld, int64_t B, int64_t D,
                            const double *obs, const double *W, const int32_t *unweighted,
                            int64_t K, double *out)
{
    for (int64_t i = 0; i < B; ++i) {
        const double *row = S + i * ld;
        for (int64_t k = 0; k < K; ++k) {
            const double *w = W + k * D;
            double acc = 0.0;
            for (int64_t j = 0; j < D; ++j) {
                double diff = fabs(row[j] - obs[j]);
                double sq = diff * diff;
                acc += unweighted[k] ? sq : w[j] * sq;
            }
            out[i * K + k] = sqrt(acc);
        }
    }
}

/* acceptance + count (elfi/methods/inference/samplers.py:223-225):
 * accepted_i = all_k(d[i,k] <= thr[k]).  Writes ascending row indices. */
int64_t oracle_accept(const double *d, int64_t B, int64_t K, const double *thr, int32_t *idx)
{
    int64_t n = 0;
    for (int64_t i = 0; i < B; ++i) {
        int ok = 1;
        for (int64_t k = 0; k < K; ++k) ok &= (d[i * K + k] <= thr[k]);
        if (ok) idx[n++] = (int32_t)i;
    }
    return n;
}

/* Other metrics that elfi.Distance hands to scipy.spatial.distance.cdist
 * (elfi/model/elfi_model.py:1016-1037).  SciPy 1.18 accumulates them left to right in fp64 like
 * 'euclidean' (pinned by tests/test_oracle.py against the installed SciPy).
 * metric: 1 sqeuclidean, 2 cityblock, 3 chebyshev, 4 minkowski(p). */
void oracle_cdist_metric(const double *S, int64_t ld, int64_t B, int64_t D, const double *obs,
                         int32_t metric, double p, double *out)
{
    for (int64_t i = 0; i < B; ++i) {
        const double *x = S + i * ld;
        double acc = 0.0;
        for (int64_t j = 0; j < D; ++j) {
            double d = x[j] - obs[j];
            if (metric == 1) acc += d * d;
            else if (metric == 2) acc += fabs(d);
            else if (metric == 3) { if (fabs(d) > acc) acc = fabs(d); }
            else acc += pow(fabs(d), p);
        }
        out[i] = (metric == 4) ? pow(acc, 1.0 / p) : acc;
    }
}

/* cdist(S, obs, 'seuclidean', V=V) as SciPy 1.18's compiled loop evaluates it: terms (d*d)/V_j,
 * even columns in one running sum and odd columns in another over the first D - D%2 columns,
 * the two added, then the last term when D is odd (pinned bit for bit against the installed SciPy
 * by tests/test_oracle.py; a single left-to-right sum differs in the last bits). */
void oracle_cdist_seuclidean(const double *S, int64_t ld, int64_t B, int64_t D, const double *obs,
                             const double *V, double *out)
{
    const int64_t D2 = D - D % 2;
    for (int64_t i = 0; i < B; ++i) {
        const double *x = S + i * ld;
        double even = 0.0, odd = 0.0;
        for (int64_t j = 0; j < D2; j += 2) {
            double d0 = x[j] - obs[j], d1 = x[j + 1] - obs[j + 1];
            even += (d0 * d0) / V[j];
            odd += (d1 * d1) / V[j + 1];
        }
        double s = even + odd;
        if (D2 < D) {
            double d = x[D2] - obs[D2];
            s += (d * d) / V[D2];
        }
        out[i] = sqrt(s);
    }
}

/* --------------------------------------------------------------------------
 * NumPy's pairwise summation (numpy/_core/src/umath/loops_utils.h.src,
 * DOUBLE_pairwise_sum), used by every np.sum/np.mean/np.var along a contiguous
 * axis -- i.e. by the reference summaries autocov (elfi/examples/ma2.py:40-59),
 * ss_mean / ss_var (elfi/examples/gauss.py:142-173).
 * ------------------------------------------------------------------------ */
static double pairwise_sum(const double *a, int64_t n, int64_t stride)
{
    if (n < 8) {
        double res = 0.0;
        for (int64_t i = 0; i < n; ++i) res += a[i * stride];
        return res;
    } else if (n <= 128) {
        double r[8];
        for (int k = 0; k < 8; ++k) r[k] = a[k * stride];
        int64_t i;
        for (i = 8; i < n - (n % 8); i += 8)
            for (int k = 0; k < 8; ++k) r[k] += a[(i + k) * stride];
        double res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
        for (; i < n; ++i) res += a[i * stride];
        return res;
    } else {
        int64_t n2 = n / 2;
        n2 -= n2 % 8;
        return pairwise_sum(a, n2, stride) + pairwise_sum(a + n2 * stride, n - n2, stride);
    }
}

/* np.add.reduce starts from the identity 0.0 and adds the pairwise sum of the run to it
 * (DOUBLE_add, IS_BINARY_REDUCE branch): only the sign of a zero sum is affected. */
static double np_sum(const double *a, int64_t n) { return 0.0 + pairwise_sum(a, n, 1); }

double oracle_pairwise_sum(const double *a, int64_t n) { return np_sum(a, n); }

/* autocov (elfi/examples/ma2.py:40-59): C_i = mean_j( x[i,j+lag] * x[i,j] ), j < n-lag.
 * NumPy materialises the product row then reduces it pairwise; same here. */
void oracle_autocov(const double *X, int64_t ld, int64_t B, int64_t n, int64_t lag, double *out)
{
    {
        double *tmp = (double *)malloc(sizeof(double) * (size_t)(n > 0 ? n : 1));
        for (int64_t i = 0; i < B; ++i) {
            const double *x = X + i * ld;
            int64_t m = n - lag;
            for (int64_t j = 0; j < m; ++j) tmp[j] = x[j + lag] * x[j];
            out[i] = np_sum(tmp, m) / (double)m;
        }
        free(tmp);
    }
}

/* ss_mean / ss_var (elfi/examples/gauss.py:142-173): np.mean(y, axis=1), np.var(y, axis=1).
 * np.var = mean(|y - mean(y)|^2) with each reduction pairwise (numpy/_core/_methods.py:_var). */
void oracle_meanvar(const double *X, int64_t ld, int64_t B, int64_t n, double *mean, double *var)
{
    {
        double *tmp = (double *)malloc(sizeof(double) * (size_t)(n > 0 ? n : 1));
        for (int64_t i = 0; i < B; ++i) {
            const double *x = X + i * ld;
            double mu = np_sum(x, n) / (double)n;
            if (mean) mean[i] = mu;
            if (var) {
                for (int64_t j = 0; j < n; ++j) {
                    double c = x[j] - mu;
                    tmp[j] = c * c;
                }
                var[i] = np_sum(tmp, n) / (double)n;
            }
        }
        free(tmp);
    }
}
