// Host build of elfi_b200/csrc/scratch_assay.cuh (test infrastructure, see
// tests/test_scratch_assay_host.py): rows simulated on the CPU from the Philox streams.
#include <cstdint>
#include <vector>

#include "../../elfi_b200/csrc/scratch_assay.cuh"

// Rows i < B of parameters P (B, 2) from the lattice init (nrows * ncols, nonzero = a cell), row
// counter offset + i: X (B, nrows, ncols, num_obs + 1) the frames as 0 / 1 (or NULL) and S
// (B, num_obs + 1) the mismatches and the final count.
extern "C" void harness_scratch_assay(const double* P, int64_t B, const uint8_t* init, int32_t nrows,
                                      int32_t ncols, int32_t num_obs, int32_t interval,
                                      uint64_t seed, uint64_t offset, uint8_t* X, double* S) {
    const int N = nrows * ncols, W = elfi::sa_words(N), F = num_obs + 1;
    const elfi::Philox ph(seed);
    std::vector<uint32_t> lat(W), prev(W);
    std::vector<uint16_t> list(N);
    for (int64_t b = 0; b < B; ++b) {
        for (int w = 0; w < W; ++w) lat[w] = 0;
        for (int s = 0; s < N; ++s)
            if (init[s]) lat[s >> 5] |= 1u << (s & 31);
        double* srow = S + b * F;
        elfi::sa_simulate_row(ph, offset + uint64_t(b), P[2 * b], P[2 * b + 1], lat.data(),
                              list.data(), nrows, ncols, num_obs, interval,
                              [&](int k, const uint32_t* cur) {
            if (k > 0) {
                int m = 0;
                for (int w = 0; w < W; ++w) m += elfi::sa_popc(cur[w] ^ prev[w]);
                srow[k - 1] = m;
            }
            for (int w = 0; w < W; ++w) prev[w] = cur[w];
            if (X)
                for (int s = 0; s < N; ++s) X[(b * N + s) * F + k] = elfi::sa_get(cur, s);
        });
        int count = 0;
        for (int w = 0; w < W; ++w) count += elfi::sa_popc(prev[w]);
        srow[num_obs] = count;
    }
}
