// Host build of elfi_b200/csrc/gnkstats.cuh (test infrastructure, see tests/test_gnk_summaries_host.py).
#include <cmath>
#include <cstdint>

#include "../../elfi_b200/csrc/gnkstats.cuh"

// sorted: S x n series, each ascending with NaN last (np.sort); picks: lo[7], hi[7], t[7];
// out: S x width, value j of series s at out[s * width + j]
extern "C" void harness_gnk_summary(const double* sorted, int64_t S, int64_t n, int32_t kind,
                                    const double* picks, double* out) {
    elfi::GnkPicks p;
    for (int q = 0; q < elfi::GNK_NQ; ++q) {
        p.lo[q] = int(picks[q]);
        p.hi[q] = int(picks[elfi::GNK_NQ + q]);
        p.t[q] = picks[2 * elfi::GNK_NQ + q];
    }
    const int w = elfi::gnk_summary_width(kind);
    for (int64_t s = 0; s < S; ++s) {
        const double* y = sorted + s * n;
        double a[elfi::GNK_NQ], b[elfi::GNK_NQ];
        for (int q = 0; q < elfi::GNK_NQ; ++q) {
            a[q] = y[p.lo[q]];
            b[q] = y[p.hi[q]];
        }
        elfi::gnk_summary(kind, p, a, b, std::isnan(y[n - 1]), out + s * w, 1);
    }
}
