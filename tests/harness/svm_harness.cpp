// Host build of elfi_b200/csrc/stable.cuh and svm.cuh (test infrastructure, see
// tests/test_svm_host.py).
#include <cmath>
#include <cstdint>

#include "../../elfi_b200/csrc/mg1.cuh"
#include "../../elfi_b200/csrc/svm.cuh"

// out[i] = levy_stable(alpha[i], beta[i], loc=eta[i], scale=kappa[i]).rvs (S0 if s0, else S1) from
// the uniforms u[i] in [0, 1) (TH) and v[i] in (0, 1] (W)
extern "C" void harness_svm_stable(const double* alpha, const double* beta, const double* kappa,
                                   const double* eta, const double* u, const double* v, int64_t n,
                                   int32_t s0, double* out) {
    for (int64_t i = 0; i < n; ++i) {
        const elfi::StableRow r = elfi::stable_row(alpha[i], beta[i], eta[i], kappa[i], s0 != 0);
        out[i] = elfi::stable_draw(r, elfi::stable_theta(u[i]), elfi::stable_expon(v[i]));
    }
}

// X (B, n) = the log-volatility of parameters P (B, 7) from the normals Z (B, n); ok[b] = the row's
// parameter check
extern "C" void harness_svm_logvol(const double* P, const double* Z, int64_t B, int32_t n,
                                   double* X, int32_t* ok) {
    for (int64_t b = 0; b < B; ++b) {
        const double* p = P + 7 * b;
        const double mu = p[4], phi = p[5], sigma = p[6];
        const double scale0 = elfi::svm_stationary_scale(phi, sigma);
        ok[b] = elfi::svm_params_ok(p[0], p[1], p[2], sigma, scale0);
        double x = elfi::svm_x0(Z[b * n], mu, scale0);
        X[b * n] = x;
        for (int j = 1; j < n; ++j) X[b * n + j] = x = elfi::svm_ar1(Z[b * n + j], x, mu, phi, sigma);
    }
}

// S (B, 2) = (kurt, skew) of the rows of X (B, n), each row sorted ascending with NaN last
extern "C" void harness_svm_summaries(const double* X, int64_t B, int32_t n, double* S) {
    for (int64_t b = 0; b < B; ++b) {
        double q[elfi::SVM_NQ];
        for (int k = 0; k < elfi::SVM_NQ; ++k)
            q[k] = elfi::mg1_quantile(n, elfi::svm_level(k), [&](int i) { return X[b * n + i]; });
        S[2 * b] = elfi::svm_kurt(q[0], q[1], q[3], q[4]);
        S[2 * b + 1] = elfi::svm_skew(q[0], q[2], q[4]);
    }
}
