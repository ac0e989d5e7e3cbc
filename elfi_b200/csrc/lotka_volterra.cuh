// lotka_volterra.cuh -- arithmetic of the stochastic Lotka-Volterra model
// (elfi/examples/lotka_volterra.py; Owen, Wilkinson & Gillespie 2015): one event of Gillespie's
// direct method, the predator-extinction time, the emission of an observation with its int32
// truncation, and the nine summaries as NumPy 2.3 computes them.  Every operation is rounded on its
// own (no FMA): leaf_add / leaf_sub / leaf_mul / gnk_div are __dadd_rn & co. on the device and
// plain operators on the host, where tests/harness/lotka_volterra_harness.cpp builds this header
// with -ffp-contract=off and checks it against NumPy.
//
// Event (lotka_volterra.py:96-120) from the counts (X, Y), an exponential E and a uniform x in
// [0, 1):
//   h1 = r1 X, h2 = (r2 X) Y, h3 = r3 Y, sum = (h1 + h2) + h3, inv = 1 / sum, dt = inv E,
//   p = h inv, reaction = (x >= p1) + (x >= p1 + p2), or the null reaction when inv is infinite;
//   R1: X + 1, R2: X - 1 and Y + 1, R3: Y - 1.  An event that leaves Y == 0 takes the time
//   time_end (so a row that starts without predators ramps linearly to its first event).
// Observation j >= 1 (lotka_volterra.py:129-138), between the last event before t_out[j] (t0, S0)
// and the first at or after it (t1, S1):  ((S1 - S0) * ((t_out[j] - t0) / (t1 - t0)) + S0) + noise,
// truncated toward zero into int32; NaN and values outside the int32 range give -2^31, as NumPy's
// float64 -> int32 cast does on x86-64.
//
// Populations are held as doubles (exact integers).  The reference keeps them in int32 until its
// event arrays switch to float64 after 20000 steps; a count changes by at most 1 per event, so it
// cannot wrap before that switch, and nothing needs emulating.
//
// Summaries of a row of n observations x (n >= 3, one leaf of NumPy's pairwise sum, LeafSum):
//   mean = sum(x) / n;  var = sum((x - mean)^2) / (n - 1);  log_var = log(var + 1)
//   autocorr_lag = sum_{i < n - lag} z[i + lag] z[i] / (n - 1),  z = (x - mean) / sqrt(var)
//   crosscorr = sum_i w_prey[i] w_pred[i] / (n - 1),  w = (x - mean) / sqrt(sum((x - mean)^2) / n)
// A constant series has sqrt(var) == 0 and gives NaN correlations, as in NumPy.
#pragma once

#include <math.h>
#include <stdint.h>

#include "hd.cuh"
#include "../../include/elfi_b200.h"
#include "gnkstats.cuh"

namespace elfi {

// observation times staged in shared memory
constexpr int LV_NOBS_MAX = ELFI_B200_LV_NOBS_MAX;
// the lag-2 autocorrelation needs one product
constexpr int LV_SUMM_NOBS_MIN = ELFI_B200_LV_SUMM_NOBS_MIN;
// one leaf of NumPy's pairwise sum (LEAF_MAX_TERMS)
constexpr int LV_SUMM_NOBS_MAX = ELFI_B200_LV_SUMM_NOBS_MAX;
constexpr int LV_NSUMM = ELFI_B200_LV_NSUMM;
constexpr double LV_INT32_LOW = -2147483649.0;   // the open interval of doubles whose truncation
constexpr double LV_INT32_HIGH = 2147483648.0;   // fits int32

ELFI_HD double lv_log(double x) { return log(x); }
ELFI_HD double lv_sqrt(double x) { return sqrt(x); }

struct LvEvent {
    double dt;      // waiting time inv * E (before the extinction rule)
    double sum;     // total hazard; the row is invalid unless sum >= 0
    int reaction;   // 0, 1, 2 or 3 (null)
};

// one event of the direct method from the counts (X, Y)
ELFI_HD LvEvent lv_event(double r1, double r2, double r3, double X, double Y, double E, double x) {
    const double h1 = leaf_mul(r1, X);
    const double h2 = leaf_mul(leaf_mul(r2, X), Y);
    const double h3 = leaf_mul(r3, Y);
    LvEvent ev;
    ev.sum = leaf_add(leaf_add(h1, h2), h3);
    const double inv = gnk_div(1.0, ev.sum);
    ev.dt = leaf_mul(inv, E);
    if (inv == INFINITY || inv == -INFINITY) {
        ev.reaction = 3;
    } else {
        const double p1 = leaf_mul(h1, inv), p2 = leaf_mul(h2, inv);
        ev.reaction = int(x >= p1) + int(x >= leaf_add(p1, p2));
    }
    return ev;
}

// the counts after a reaction
ELFI_HD void lv_apply(int reaction, double& X, double& Y) {
    if (reaction == 0) {
        X = leaf_add(X, 1.0);
    } else if (reaction == 1) {
        X = leaf_sub(X, 1.0);
        Y = leaf_add(Y, 1.0);
    } else if (reaction == 2) {
        Y = leaf_sub(Y, 1.0);
    }
}

// the time of an event that leaves Y predators: time_end once they are gone
ELFI_HD double lv_event_time(double t_prev, double dt, double Y, double time_end) {
    return Y == 0.0 ? time_end : leaf_add(t_prev, dt);
}

// float64 -> int32 as NumPy casts it on x86-64 (cvttsd2si), returned as a double
ELFI_HD double lv_to_int32(double v) {
    if (!(v > LV_INT32_LOW && v < LV_INT32_HIGH)) return -2147483648.0;
    return trunc(v);
}

// observation at t_out between the events (t0, s0) and (t1, s1), plus noise, truncated
ELFI_HD double lv_emit(double t_out, double t0, double s0, double t1, double s1, double noise) {
    const double frac = gnk_div(leaf_sub(t_out, t0), leaf_sub(t1, t0));
    return lv_to_int32(leaf_add(leaf_add(leaf_mul(leaf_sub(s1, s0), frac), s0), noise));
}

// The state of one row between events.
struct LvState {
    double r1, r2, r3, sigma;
    double t, X, Y;   // the last event
    uint32_t k;       // events run
    int j;            // next observation
};

ELFI_HD bool lv_count_ok(double c) { return c >= 0.0 && c < 2147483648.0; }

// Starts a row from p = (r1, r2, r3, prey0, predator0, sigma); observation 0 is (X, Y).  Returns
// false for parameters the reference rejects (or whose arithmetic stops meaning anything).
ELFI_HD bool lv_init(LvState& s, const double* p) {
    s.r1 = p[0];
    s.r2 = p[1];
    s.r3 = p[2];
    s.X = floor(p[3]);
    s.Y = floor(p[4]);
    s.sigma = p[5];
    s.t = 0.0;
    s.k = 0;
    s.j = 1;
    return s.r1 >= 0.0 && s.r2 >= 0.0 && s.r3 >= 0.0 && s.sigma >= 0.0 && lv_count_ok(s.X) &&
           lv_count_ok(s.Y);
}

// One event of the row from its exponential E and uniform u.  Every observation the event
// reaches (t_out[j] <= its time) is passed to emit(j, prey, predators); normals(j, n0, n1) gives
// its two standard normals, asked for only when sigma != 0.  Returns false, leaving the state
// alone, when the total hazard is negative or NaN.
template <class Normals, class Emit>
ELFI_HD bool lv_advance(LvState& s, double E, double u, const double* t_out, int n_obs,
                        double time_end, const Normals& normals, const Emit& emit) {
    const LvEvent ev = lv_event(s.r1, s.r2, s.r3, s.X, s.Y, E, u);
    if (!(ev.sum >= 0.0)) return false;
    double X1 = s.X, Y1 = s.Y;
    lv_apply(ev.reaction, X1, Y1);
    const double t1 = lv_event_time(s.t, ev.dt, Y1, time_end);
    for (; s.j < n_obs && t1 >= t_out[s.j]; ++s.j) {
        double n0 = 0.0, n1 = 0.0;
        if (s.sigma != 0.0) {
            normals(s.j, n0, n1);
            n0 = leaf_mul(s.sigma, n0);
            n1 = leaf_mul(s.sigma, n1);
        }
        emit(s.j, lv_emit(t_out[s.j], s.t, s.X, t1, X1, n0),
             lv_emit(t_out[s.j], s.t, s.Y, t1, Y1, n1));
    }
    s.t = t1;
    s.X = X1;
    s.Y = Y1;
    ++s.k;
    return true;
}

// a row is complete once it has reached time_end (then every observation has been emitted);
// short of it after max_events events, or with a NaN time, its observations are NaN
ELFI_HD bool lv_running(const LvState& s, double time_end, uint32_t max_events) {
    return s.t < time_end && s.k < max_events;
}
ELFI_HD bool lv_complete(const LvState& s, double time_end, int n_obs) {
    return s.t >= time_end && s.j == n_obs;
}

// sum_{j < m} f(j) in NumPy's pairwise order (one leaf, m <= 128)
template <int J, class F>
ELFI_HD void lv_push8(LeafSum& s, int j0, int m, const F& f) {
    if (j0 + J < m) s.template push<J>(j0 + J, f(j0 + J));
    if constexpr (J + 1 < 8) lv_push8<J + 1>(s, j0, m, f);
}
template <class F>
ELFI_HD double lv_leaf_sum(int m, const F& f) {
    LeafSum s;
    s.begin(m);
    for (int j0 = 0; j0 < m; j0 += 8) lv_push8<0>(s, j0, m, f);
    return s.finish(m);
}

// the nine summaries of a row: x(i, s) is observation i of species s (0 prey, 1 predators);
// out[0..8] = prey_mean, pred_mean, prey_log_var, pred_log_var, prey_autocorr_1, pred_autocorr_1,
// prey_autocorr_2, pred_autocorr_2, crosscorr
template <class Get>
ELFI_HD void lv_summaries(int n, const Get& x, double* out) {
    const double dn = double(n), dn1 = double(n - 1);
    double mean[2], sd1[2], sd0[2];
    for (int s = 0; s < 2; ++s) {
        mean[s] = gnk_div(lv_leaf_sum(n, [&](int i) { return x(i, s); }), dn);
        const double m = mean[s];
        const double ss = lv_leaf_sum(n, [&](int i) {
            const double c = leaf_sub(x(i, s), m);
            return leaf_mul(c, c);
        });
        const double var1 = gnk_div(ss, dn1);
        sd1[s] = lv_sqrt(var1);
        sd0[s] = lv_sqrt(gnk_div(ss, dn));
        out[s] = mean[s];
        out[2 + s] = lv_log(leaf_add(var1, 1.0));
    }
    for (int lag = 1; lag <= 2; ++lag) {
        for (int s = 0; s < 2; ++s) {
            const double m = mean[s], sd = sd1[s];
            const double c = lv_leaf_sum(n - lag, [&](int i) {
                return leaf_mul(gnk_div(leaf_sub(x(i + lag, s), m), sd),
                                gnk_div(leaf_sub(x(i, s), m), sd));
            });
            out[2 + 2 * lag + s] = gnk_div(c, dn1);
        }
    }
    const double c = lv_leaf_sum(n, [&](int i) {
        return leaf_mul(gnk_div(leaf_sub(x(i, 0), mean[0]), sd0[0]),
                        gnk_div(leaf_sub(x(i, 1), mean[1]), sd0[1]));
    });
    out[8] = gnk_div(c, dn1);
}

}  // namespace elfi
