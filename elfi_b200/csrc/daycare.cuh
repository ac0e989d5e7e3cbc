// daycare.cuh -- arithmetic of the day care model (elfi/examples/daycare.py; Numminen et al. 2013):
// one transition of Gillespie's direct method in one day care centre (DCC), the four summaries of
// its observed children, and the sorted-L1 distance of a row.  Every operation is rounded on its
// own (leaf_add / leaf_mul / gnk_div), so tests/harness/daycare_harness.cpp builds this header for
// the host with -ffp-contract=off and tests/daycare_replay.py restates it in NumPy bit for bit.
//
// State of a DCC: one 64-bit strain mask per child, and per strain s the number c_s of carriers and
// the numerator num_s = sum over the carriers i of s of L / n_i, where n_i is the number of strains
// child i carries and L = lcm(1 .. n_strains).  So E_s = num_s / L (daycare.py:102-103) is held as
// an exact integer: a transition changes only the numerators of the flipped child's strains, and
// nothing drifts however many transitions a row takes.  double(num_s) is exact while
// L * n_ind < 2^53 (the defaults: 7.7e15); beyond that it is rounded once.
//
// Hazards (daycare.py:106-118), with nf = 1 / (n_ind - 1):
//   h_s = ((t1 E_s) nf + 1e-9) + t2 f_s         a non-carrier of s who carries nothing
//   t3 h_s                                     a non-carrier of s who carries another strain
//   1                                          a carrier of s (gamma)
// Per strain the weight is W_s = c_s + h_s (u + t3 (n_ind - u - c_s)), u the children carrying
// nothing, and the total H = sum_s W_s in strain order.  The waiting time is (1 / H) E.
// Selection from a uniform x in [0, 1): target = x H; the strain is the first with target below
// the running sum of W (the last strain with W > 0 if rounding leaves none); within it, in the
// order recoveries, infections of children carrying nothing, infections of children carrying
// another strain, the category and then the child (in index order) whose slot holds the rest of the
// target.  The reference walks the same cells in child-major order instead; the law is the same.
#pragma once

#include <math.h>
#include <stdint.h>

#include "hd.cuh"
#include "../../include/elfi_b200.h"
#include "lotka_volterra.cuh"   // lv_leaf_sum: NumPy's pairwise order for <= 128 terms

namespace elfi {

constexpr int DC_DCC_MAX = ELFI_B200_DC_DCC_MAX;        // one lane per DCC
// num_s * 64 stays within int64 for n_strains <= 40
constexpr int DC_IND_MAX = ELFI_B200_DC_IND_MAX;
constexpr int DC_STRAINS_MAX = ELFI_B200_DC_STRAINS_MAX;    // lcm(1 .. 40) = 5.3e15 < 2^53
constexpr int DC_NSUMM = ELFI_B200_DC_NSUMM;           // Shannon, n_strains, prevalence, multi
// n_ss * n_dcc of the distance (one pairwise leaf)
constexpr int DC_DIST_TERMS_MAX = ELFI_B200_DC_DIST_TERMS_MAX;
constexpr double DC_EVENTS_MAX = 4294967295.0;   // transitions per row: the stream's event word

ELFI_HD int dc_popc(uint64_t m) {
#if defined(__CUDA_ARCH__)
    return __popcll(m);
#else
    return __builtin_popcountll(m);
#endif
}

ELFI_HD double dc_log(double x) { return log(x); }

// lcm(1 .. n), n <= DC_STRAINS_MAX
inline int64_t dc_lcm(int n) {
    int64_t L = 1;
    for (int k = 2; k <= n; ++k) {
        int64_t a = L, b = k;
        while (b) {
            const int64_t r = a % b;
            a = b;
            b = r;
        }
        L = L / a * k;
    }
    return L;
}

// Whether a row runs: t1, t2, t3 finite and >= 0, and time_end times the largest total hazard a
// DCC can reach below DC_EVENTS_MAX, so that the expected number of transitions of every DCC is
// bounded by the event word.  A non-carrier's E_s / (n_ind - 1) is at most 1, so a cell's hazard is
// at most max(1, max(1, t3) (t1 + 1e-9 + t2 f_max)), f_max the largest community frequency (finite
// and >= 0, checked by the caller), and the total is at most n_ind n_strains times that.
ELFI_HD bool dc_row_ok(double t1, double t2, double t3, double f_max, int n_ind, int n_strains,
                       double time_end) {
    if (!(t1 >= 0.0 && t1 < INFINITY && t2 >= 0.0 && t2 < INFINITY && t3 >= 0.0 && t3 < INFINITY))
        return false;
    const double h = (t1 + 1e-9) + t2 * f_max;
    const double cell = fmax(1.0, fmax(1.0, t3) * h);
    return time_end * double(n_ind) * double(n_strains) * cell < DC_EVENTS_MAX;
}

// The parameters of one row and the model's constants.
struct DcParams {
    double t1, t2, t3, nf, Ld;   // nf = 1 / (n_ind - 1), Ld = double(L)
    const double* f;             // freq_strains_commun (n_strains)
    const int64_t* Lk;           // Lk[k] = L / k, 1 <= k <= n_strains
    int n_ind, n_strains;
};

// One DCC's state; element i of a field is at [i * stride] (the kernel interleaves the lanes).
struct DcState {
    uint64_t* mask;   // (n_ind)
    int64_t* num;     // (n_strains)
    int32_t* cnt;     // (n_strains)
    int stride;
    int n_free;       // children carrying nothing
};

ELFI_HD void dc_clear(DcState& st, const DcParams& p) {
    for (int i = 0; i < p.n_ind; ++i) st.mask[i * st.stride] = 0;
    for (int s = 0; s < p.n_strains; ++s) {
        st.num[s * st.stride] = 0;
        st.cnt[s * st.stride] = 0;
    }
    st.n_free = p.n_ind;
}

// the hazard of a non-carrier of s who carries nothing
ELFI_HD double dc_h(const DcParams& p, const DcState& st, int s) {
    const double E = gnk_div(double(st.num[s * st.stride]), p.Ld);
    return leaf_add(leaf_add(leaf_mul(leaf_mul(p.t1, E), p.nf), 1e-9), leaf_mul(p.t2, p.f[s]));
}

// the weight W_s of strain s given h = dc_h(s)
ELFI_HD double dc_weight(const DcParams& p, const DcState& st, int s, double h) {
    const int c = st.cnt[s * st.stride];
    const int m = p.n_ind - st.n_free - c;
    return leaf_add(double(c), leaf_mul(h, leaf_add(double(st.n_free), leaf_mul(p.t3, double(m)))));
}

ELFI_HD double dc_total(const DcParams& p, const DcState& st) {
    double H = 0.0;
    for (int s = 0; s < p.n_strains; ++s) H = leaf_add(H, dc_weight(p, st, s, dc_h(p, st, s)));
    return H;
}

// floor(q) clamped to [0, n - 1]
ELFI_HD int dc_slot(double q, int n) {
    if (!(q > 0.0)) return 0;
    return q >= double(n - 1) ? n - 1 : int(q);
}

// the j-th child (index order) of category cat for strain s: 0 carriers of s, 1 children carrying
// nothing, 2 children carrying another strain but not s
ELFI_HD int dc_child(const DcParams& p, const DcState& st, int cat, int s, int j) {
    const uint64_t bit = uint64_t(1) << s;
    int last = 0;
    for (int i = 0; i < p.n_ind; ++i) {
        const uint64_t m = st.mask[i * st.stride];
        const bool in = cat == 0 ? (m & bit) != 0 : cat == 1 ? m == 0 : (m != 0 && !(m & bit));
        if (in) {
            if (j == 0) return i;
            --j;
            last = i;
        }
    }
    return last;
}

struct DcPick {
    int child, strain;
};

// The transition a uniform x in [0, 1) selects, H = dc_total.  strain = child = -1 when no strain
// has a positive weight (which rows that pass dc_row_ok never reach: h_s >= 1e-9, so a child
// carrying nothing or a carrier always gives some W_s > 0).
ELFI_HD DcPick dc_pick(const DcParams& p, const DcState& st, double H, double x) {
    const double target = leaf_mul(x, H);
    double cum = 0.0, start = 0.0;
    int strain = -1;
    for (int s = 0; s < p.n_strains; ++s) {
        const double W = dc_weight(p, st, s, dc_h(p, st, s));
        const double next = leaf_add(cum, W);
        if (W > 0.0) {
            strain = s;
            start = cum;
            if (target < next) break;
        }
        cum = next;
    }
    DcPick out;
    out.strain = out.child = -1;
    if (strain < 0) return out;
    const int s = strain;
    const double h = dc_h(p, st, s);
    const int c = st.cnt[s * st.stride];
    const int m = p.n_ind - st.n_free - c;
    const double w0 = double(c), w1 = leaf_mul(h, double(st.n_free));
    const double th = leaf_mul(p.t3, h), w2 = leaf_mul(th, double(m));
    double r = leaf_sub(target, start);
    if (!(r > 0.0)) r = 0.0;
    out.strain = s;
    if (w0 > 0.0 && (r < w0 || !(w1 > 0.0 || w2 > 0.0))) {
        out.child = dc_child(p, st, 0, s, dc_slot(r, c));
        return out;
    }
    r = leaf_sub(r, w0);
    if (!(r > 0.0)) r = 0.0;
    if (w1 > 0.0 && (r < w1 || !(w2 > 0.0))) {
        out.child = dc_child(p, st, 1, s, dc_slot(gnk_div(r, h), st.n_free));
        return out;
    }
    r = leaf_sub(r, w1);
    if (!(r > 0.0)) r = 0.0;
    out.child = dc_child(p, st, 2, s, dc_slot(gnk_div(r, th), m));
    return out;
}

// flips strain s of child i
ELFI_HD void dc_flip(const DcParams& p, DcState& st, int i, int s) {
    uint64_t m = st.mask[i * st.stride];
    int n = dc_popc(m);
    for (uint64_t b = m; b; b &= b - 1) st.num[dc_popc((b & (~b + 1)) - 1) * st.stride] -= p.Lk[n];
    const uint64_t bit = uint64_t(1) << s;
    const bool was = (m & bit) != 0;
    st.cnt[s * st.stride] += was ? -1 : 1;
    if (m == 0) --st.n_free;
    m ^= bit;
    if (m == 0) ++st.n_free;
    st.mask[i * st.stride] = m;
    n = dc_popc(m);
    for (uint64_t b = m; b; b &= b - 1) st.num[dc_popc((b & (~b + 1)) - 1) * st.stride] += p.Lk[n];
}

// One transition from the exponential E and the uniform x in [0, 1); returns the waiting time, or
// NaN (leaving the state alone) when dc_pick finds no transition.
ELFI_HD double dc_step(const DcParams& p, DcState& st, double E, double x) {
    const double H = dc_total(p, st);
    const DcPick k = dc_pick(p, st, H, x);
    if (k.strain < 0) return NAN;
    dc_flip(p, st, k.child, k.strain);
    return leaf_mul(gnk_div(1.0, H), E);
}

// The four summaries (daycare.py:199-275) of a DCC whose observed children have the strain masks
// obs(0 .. n_obs - 1): out[0] Shannon, out[k * step] for n_strains, prevalence and multi.
template <class Obs>
ELFI_HD void dc_summaries(int n_obs, int n_strains, const Obs& obs, double* out, int64_t step) {
    int cnt[64];
    for (int s = 0; s < n_strains; ++s) cnt[s] = 0;
    uint64_t any = 0;
    int infected = 0, multi = 0, total = 0;
    for (int i = 0; i < n_obs; ++i) {
        const uint64_t m = obs(i);
        const int n = dc_popc(m);
        any |= m;
        infected += m != 0;
        multi += n > 1;
        total += n;
        for (uint64_t b = m; b; b &= b - 1) ++cnt[dc_popc((b & (~b + 1)) - 1)];
    }
    // proportions, nan_to_num (0 / 0 -> 0), zeros -> 1, then -sum(p log p)
    const double sum = lv_leaf_sum(n_strains, [&](int s) {
        const double q = total > 0 ? gnk_div(double(cnt[s]), double(total)) : 0.0;
        const double pr = q == 0.0 ? 1.0 : q;
        return leaf_mul(pr, dc_log(pr));
    });
    out[0] = -sum;
    out[step] = double(dc_popc(any));
    out[2 * step] = gnk_div(double(infected), double(n_obs));
    out[3 * step] = gnk_div(double(multi), double(n_obs));
}

// NumPy's sort order: ascending, NaN last
ELFI_HD bool dc_before(double a, double b) { return a < b || (b != b && a == a); }

// The distance of daycare.py:278-312 for one row: s(k, c) is summary k of DCC c; obs_max (n_ss)
// the observed maxima with 0 replaced by 1 and y (n_ss, n_dcc) the observed values divided by them
// and sorted.  NumPy sums |x - y| over (summary, DCC) as one pairwise sum when the batch has one
// row (single), else as one pairwise sum per summary, those added in order.
template <class Get>
ELFI_HD double dc_distance(int n_ss, int n_dcc, const Get& s, const double* obs_max,
                           const double* y, bool single) {
    double terms[DC_DIST_TERMS_MAX];
    for (int k = 0; k < n_ss; ++k) {
        double* x = terms + k * n_dcc;
        for (int c = 0; c < n_dcc; ++c) {
            const double v = gnk_div(s(k, c), obs_max[k]);
            int j = c;
            for (; j > 0 && dc_before(v, x[j - 1]); --j) x[j] = x[j - 1];
            x[j] = v;
        }
        for (int c = 0; c < n_dcc; ++c) x[c] = fabs(leaf_sub(x[c], y[k * n_dcc + c]));
    }
    double total;
    if (single) {
        total = lv_leaf_sum(n_ss * n_dcc, [&](int j) { return terms[j]; });
    } else {
        total = 0.0;
        for (int k = 0; k < n_ss; ++k) {
            const double part = lv_leaf_sum(n_dcc, [&](int j) { return terms[k * n_dcc + j]; });
            total = k == 0 ? part : leaf_add(total, part);
        }
    }
    return gnk_div(total, double(n_ss * n_dcc));
}

}  // namespace elfi
