// bdm.cuh -- arithmetic of the birth-death-mutation (BDM) model of tuberculosis transmission
// (Tanaka et al. 2006) as elfi/examples/cpp/bdm.cpp runs it with --mode 1: one event of the
// process, the end of a row, and the summaries T1 and T2 of elfi/examples/bdm.py as NumPy computes
// them.  Every operation is rounded on its own (no FMA): leaf_add / leaf_mul / gnk_div are
// __dadd_rn & co. on the device and plain operators on the host, where
// tests/harness/bdm_harness.cpp builds this header with -ffp-contract=off and checks it against
// the reference executable and against NumPy.
//
// A row of parameters (alpha, delta, tau) and population bound N keeps N cluster counts c[0..N),
// at first c[0] = 1 and the rest 0, pop = 1 and end = 1 (every nonzero count lies below end).
// While 0 < pop < N + 1, one event draws u then v, both in [0, 1):
//   event: total = ((0.0 + alpha) + delta) + tau; the first k whose running sum of
//          (alpha, delta, tau) exceeds u * total (0 birth, 1 death, 2 mutation);
//   cluster: the first j < end with (double)(c[0] + ... + c[j]) > v * pop;
//   birth: c[j] += 1, pop += 1;  death: c[j] -= 1, pop -= 1;
//   mutation, only when c[j] > 1: c[j] -= 1 and the first zero count of c[0..N) becomes 1.
// With u < 1, u * total rounds below total (and v * pop below pop), so both draws always find an
// index.  A row that ends on a birth (pop == N + 1) has that birth undone.
//
// Summaries of counts c[0..N) and the T2 argument n:
//   T1 = count(c > 0) / sum(c)  (0 / 0 is NaN: an extinct row)
//   T2 = 1 - sum_j (c_j / n)^2, the sum in NumPy's pairwise order.
#pragma once

#include <math.h>
#include <stdint.h>

#include "gnkstats.cuh"
#include "hd.cuh"
#include "../../include/elfi_b200.h"
#include "leafsum.cuh"
#include "treesum.cuh"

namespace elfi {

// a count stays below N + 2 <= 2^16 (uint16 in shared memory)
constexpr int BDM_N_MAX = ELFI_B200_BDM_N_MAX;
constexpr int BDM_NSUMM = ELFI_B200_BDM_NSUMM;          // T1, T2
constexpr int BDM_PW_DEPTH = 4;       // TreeSum<4> sums up to 1928 terms in NumPy's order

// The state of one row between events; the counts are c[j * stride] in the caller's storage.
struct BdmState {
    double alpha, delta, tau, total;
    int N, pop, end;
    int event, cluster;    // the last event and its cluster
    uint32_t k;            // events run
};

// Starts a row: false for rates the reference cannot run (negative, NaN or infinite, or a total
// that is 0 or overflows; the executable throws for a zero total).
template <class C>
ELFI_HD bool bdm_init(BdmState& s, double alpha, double delta, double tau, int N, C* c,
                      int stride) {
    s.alpha = alpha;
    s.delta = delta;
    s.tau = tau;
    s.total = leaf_add(leaf_add(leaf_add(0.0, alpha), delta), tau);
    s.N = N;
    s.pop = 1;
    s.end = 1;
    s.event = 0;
    s.cluster = 0;
    s.k = 0;
    for (int j = 0; j < N; ++j) c[j * stride] = 0;
    c[0] = 1;
    return alpha >= 0.0 && alpha < INFINITY && delta >= 0.0 && delta < INFINITY && tau >= 0.0 &&
           tau < INFINITY && s.total > 0.0 && s.total < INFINITY;
}

ELFI_HD bool bdm_running(const BdmState& s) { return s.pop > 0 && s.pop < s.N + 1; }

// the event drawn by u in [0, 1)
ELFI_HD int bdm_event(const BdmState& s, double u) {
    const double x = leaf_mul(u, s.total);
    double cum = leaf_add(0.0, s.alpha);
    if (cum > x) return 0;
    cum = leaf_add(cum, s.delta);
    if (cum > x) return 1;
    return 2;
}

// the cluster drawn by v in [0, 1)
template <class C>
ELFI_HD int bdm_cluster(const BdmState& s, double v, const C* c, int stride) {
    const double x = leaf_mul(v, double(s.pop));
    int cum = 0;
    for (int j = 0; j < s.end; ++j) {
        cum += int(c[j * stride]);
        if (double(cum) > x) return j;
    }
    return s.end - 1;   // not reached: the counts below end sum to pop > x
}

// One event from its uniforms u (event) and v (cluster).
template <class C>
ELFI_HD void bdm_step(BdmState& s, double u, double v, C* c, int stride) {
    const int e = bdm_event(s, u);
    const int j = bdm_cluster(s, v, c, stride);
    C* cj = c + j * stride;
    if (e == 0) {
        *cj = C(*cj + 1);
        ++s.pop;
    } else if (e == 1) {
        *cj = C(*cj - 1);
        --s.pop;
    } else if (*cj > 1) {
        *cj = C(*cj - 1);
        // a zero exists: c[j] > 1 leaves at most pop - 1 < N counts nonzero
        int z = 0;
        while (z < s.N - 1 && c[z * stride] != 0) ++z;
        c[z * stride] = 1;
        if (z + 1 > s.end) s.end = z + 1;
    }
    s.event = e;
    s.cluster = j;
    ++s.k;
}

// The end of a finished row: a last birth (the one that reached N + 1) is undone.
template <class C>
ELFI_HD void bdm_finish(BdmState& s, C* c, int stride) {
    if (s.event == 0) {
        C* cj = c + s.cluster * stride;
        *cj = C(*cj - 1);
        --s.pop;
    }
}

// sum_{j < m} f(j) in NumPy's pairwise order
template <int K, class F>
ELFI_HD void bdm_push8(TreeSum<BDM_PW_DEPTH>& t, int j0, int m, const F& f) {
    if (j0 + K < m) t.template push<K>(j0 + K, f(j0 + K));
    if constexpr (K + 1 < 8) bdm_push8<K + 1>(t, j0, m, f);
}

// T1 and T2 of the N counts count(j) (integers >= 0) with T2's argument n.
template <class Get>
ELFI_HD void bdm_summaries(int N, double n, const Get& count, double* out) {
    int64_t nonzero = 0, sum = 0;
    TreeSum<BDM_PW_DEPTH> t;
    t.begin(N);
    for (int j0 = 0; j0 < N; j0 += 8) {
        bdm_push8<0>(t, j0, N, [&](int j) {
            const int cj = int(count(j));
            nonzero += cj > 0;
            sum += cj;
            const double q = gnk_div(double(cj), n);
            return leaf_mul(q, q);
        });
    }
    out[0] = gnk_div(double(nonzero), double(sum));
    out[1] = leaf_sub(1.0, t.finish(N));
}

}  // namespace elfi
