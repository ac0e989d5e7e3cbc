// Host build of elfi_b200/csrc/daycare.cuh (test infrastructure, see tests/test_daycare_host.py).
#include <cmath>
#include <cstdint>
#include <vector>

#include "../../elfi_b200/csrc/daycare.cuh"

namespace {

struct Dcc {
    std::vector<uint64_t> mask;
    std::vector<int64_t> num, Lk;
    std::vector<int32_t> cnt;
    elfi::DcParams p;
    elfi::DcState st;

    // the state of the given strain masks, built by flipping their bits one by one from empty
    Dcc(const uint64_t* masks, int n_ind, int n_strains, const double* prm, const double* f)
        : mask(n_ind), num(n_strains), Lk(n_strains + 1), cnt(n_strains) {
        const int64_t L = elfi::dc_lcm(n_strains);
        for (int k = 1; k <= n_strains; ++k) Lk[k] = L / k;
        p.t1 = prm[0];
        p.t2 = prm[1];
        p.t3 = prm[2];
        p.nf = 1.0 / double(n_ind - 1);
        p.Ld = double(L);
        p.f = f;
        p.Lk = Lk.data();
        p.n_ind = n_ind;
        p.n_strains = n_strains;
        st.mask = mask.data();
        st.num = num.data();
        st.cnt = cnt.data();
        st.stride = 1;
        elfi::dc_clear(st, p);
        for (int i = 0; i < n_ind; ++i)
            for (int s = 0; s < n_strains; ++s)
                if ((masks[i] >> s) & 1) elfi::dc_flip(p, st, i, s);
    }
};

}  // namespace

// the total hazard of a state, its h_s (n_strains) and its numerators num_s (n_strains)
extern "C" double harness_dc_total(const uint64_t* masks, int32_t n_ind, int32_t n_strains,
                                   const double* prm, const double* f, double* h, int64_t* num) {
    Dcc d(masks, n_ind, n_strains, prm, f);
    for (int s = 0; s < n_strains; ++s) {
        h[s] = elfi::dc_h(d.p, d.st, s);
        num[s] = d.num[s];
    }
    return elfi::dc_total(d.p, d.st);
}

// whether rows of parameters prm (n, 3) run
extern "C" void harness_dc_row_ok(const double* prm, int64_t n, double f_max, int32_t n_ind,
                                  int32_t n_strains, double time_end, int32_t* ok) {
    for (int64_t j = 0; j < n; ++j)
        ok[j] = elfi::dc_row_ok(prm[3 * j], prm[3 * j + 1], prm[3 * j + 2], f_max, n_ind,
                                n_strains, time_end);
}

// the transitions (child * n_strains + strain, or -1 for none) the uniforms x (n) select
extern "C" void harness_dc_pick(const uint64_t* masks, int32_t n_ind, int32_t n_strains,
                                const double* prm, const double* f, const double* x, int64_t n,
                                int64_t* cell) {
    Dcc d(masks, n_ind, n_strains, prm, f);
    const double H = elfi::dc_total(d.p, d.st);
    for (int64_t j = 0; j < n; ++j) {
        const elfi::DcPick k = elfi::dc_pick(d.p, d.st, H, x[j]);
        cell[j] = k.strain < 0 ? -1 : int64_t(k.child) * n_strains + k.strain;
    }
}

// n_steps transitions from the draws E, x; returns the final masks and the numerators
extern "C" void harness_dc_run(uint64_t* masks, int32_t n_ind, int32_t n_strains,
                               const double* prm, const double* f, const double* E,
                               const double* x, int64_t n_steps, double* dt, int64_t* num) {
    Dcc d(masks, n_ind, n_strains, prm, f);
    for (int64_t k = 0; k < n_steps; ++k) dt[k] = elfi::dc_step(d.p, d.st, E[k], x[k]);
    for (int i = 0; i < n_ind; ++i) masks[i] = d.mask[i];
    for (int s = 0; s < n_strains; ++s) num[s] = d.num[s];
}

// summaries of n_rows DCCs of n_obs children: S[j * n_rows + r]
extern "C" void harness_dc_summaries(const uint64_t* masks, int64_t n_rows, int32_t n_obs,
                                     int32_t n_strains, double* S) {
    for (int64_t r = 0; r < n_rows; ++r)
        elfi::dc_summaries(n_obs, n_strains, [&](int i) { return masks[r * n_obs + i]; }, S + r,
                           n_rows);
}

// distances of B rows S[b * n_ss * n_dcc + k * n_dcc + c]
extern "C" void harness_dc_distance(const double* S, int64_t B, int32_t n_ss, int32_t n_dcc,
                                    const double* obs_max, const double* y, double* d) {
    for (int64_t b = 0; b < B; ++b) {
        const double* s = S + b * n_ss * n_dcc;
        d[b] = elfi::dc_distance(n_ss, n_dcc, [&](int k, int c) { return s[k * n_dcc + c]; },
                                 obs_max, y, B == 1);
    }
}
