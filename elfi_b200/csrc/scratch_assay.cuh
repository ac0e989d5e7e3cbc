// scratch_assay.cuh -- the law of the scratch assay simulator of elfi/examples/scratch_assay.py
// (Johnston et al. 2014) in throughput mode, shared by the device kernel (scratch_assay.cu) and the
// host build of the tests (tests/harness/scratch_assay_harness.cpp).  Every random decision is an
// integer or an exact fp64 comparison, so a NumPy replay of the streams (tests/scratch_assay_replay.py)
// reproduces every lattice bit.
//
// The lattice of nrows x ncols sites (N = nrows * ncols <= SA_SITES_MAX) is bit-packed row-major:
// site s = r * ncols + c is bit s & 31 of word s >> 5.  The law is the reference's cell_sim:
//   * Snapshot at the start of each iteration t: num_cells (n) and the list of occupied sites in
//     row-major order (np.where), taken once.  Motility updates a moved cell's list entry;
//     proliferation uses the same list after motility, so daughter cells are not in it and n is
//     still the count at the start of the iteration.
//   * Candidate slots: each phase (f = 0 motility, f = 1 proliferation) has n slots.  Slot s picks
//     a list index with replacement and is kept when u < pm (pp), u uniform on [0, 1).  Kept slots
//     are applied strictly in slot order: a cell may move twice in one iteration, and into a site
//     vacated earlier in the same iteration.
//   * Moving: one of the 4 directions (0: row + 1, 1: row - 1, 2: col + 1, 3: col - 1) uniformly,
//     the target clamped to the grid.  Motility moves only onto an empty site (a clamped move onto
//     the cell's own site is no move); proliferation sets the target site whether or not it is
//     occupied (so the order of its kept slots does not matter).
//   * A full lattice (n == N at the start of an iteration) does nothing in that iteration, and
//     records no observation: the reference's frames start as ones, i.e. full, so every later
//     frame is the full lattice.  The simulation may stop there.
//   * Observations: frame 0 is the initial lattice, frame k the lattice after iteration
//     k * interval - 1, k = 1 .. num_obs.  The summaries are the mismatches
//     popcount(frame_{k-1} XOR frame_k), k = 1 .. num_obs, then the popcount of frame num_obs.
//   * Parameters: pm or pp >= 1 keeps every slot; <= 0 or NaN keeps none (this is u < p), so no
//     parameter gives a NaN row.
//
// Streams (Philox4x32-10 keyed by the seed, philox.cuh), row = offset + i: slot s of phase f in
// iteration t uses the block (x, y, z, w) of counter (row, row >> 32, 2 t + f, SALT_SCRATCH + s):
//   kept       1 - u01(x, y) < p           (u01 reads x and the high 21 bits of y)
//   index      ((z << 32 | w) * n) >> 64   (a list index in [0, n); bias at most n / 2^64)
//   direction  y & 3                       (two bits of y that u01 does not read)
// So every draw is a pure function of (seed, offset + i, t, f, s), whatever the batch split.  (The
// reference draws all indices of a phase, then all uniforms, then one direction per kept slot.)
#pragma once

#include <stdint.h>

#include "hd.cuh"
#include "../../include/elfi_b200.h"
#include "leafsum.cuh"
#include "philox.cuh"

namespace elfi {

constexpr uint32_t SALT_SCRATCH = 0x53434131u;   // "SCA1"; slot s adds s (s < SA_SITES_MAX)
// lattice sites: list entries fit uint16
constexpr int SA_SITES_MAX = ELFI_B200_SA_SITES_MAX;
constexpr int SA_WORDS_MAX = SA_SITES_MAX / 32;
constexpr int SA_NPARAMS = 2;                    // pm, pp

ELFI_HD int sa_words(int nsites) { return (nsites + 31) >> 5; }

ELFI_HD int sa_popc(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return __popc(x);
#else
    return __builtin_popcount(x);
#endif
}

// index of the lowest set bit (x != 0)
ELFI_HD int sa_ctz(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return __ffs(x) - 1;
#else
    return __builtin_ctz(x);
#endif
}

// high 64 bits of a * b
ELFI_HD uint64_t sa_mulhi64(uint64_t a, uint64_t b) {
#if defined(__CUDA_ARCH__)
    return __umul64hi(a, b);
#else
    return uint64_t((unsigned __int128)a * b >> 64);
#endif
}

struct SaSlot {
    bool kept;
    int index;    // list index in [0, n)
    int dir;      // 0 .. 3
};

// slot s of phase f (0 motility, 1 proliferation) in iteration t, n cells at its start, keep
// probability p
ELFI_HD SaSlot sa_slot(const Philox& ph, uint64_t row, int t, int f, int s, int n, double p) {
    const PhiloxWords r = ph(uint32_t(row), uint32_t(row >> 32), 2u * uint32_t(t) + uint32_t(f),
                             SALT_SCRATCH + uint32_t(s));
    SaSlot out;
    out.kept = 1.0 - u01(r.x, r.y) < p;
    out.index = int(sa_mulhi64((uint64_t(r.z) << 32) | r.w, uint64_t(n)));
    out.dir = int(r.y & 3u);
    return out;
}

// the site a move from `site` in direction dir reaches, clamped to the grid
ELFI_HD int sa_target(int site, int dir, int nrows, int ncols) {
    int r = site / ncols, c = site - r * ncols;
    if (dir == 0) r = r + 1 < nrows ? r + 1 : r;
    else if (dir == 1) r = r > 0 ? r - 1 : r;
    else if (dir == 2) c = c + 1 < ncols ? c + 1 : c;
    else c = c > 0 ? c - 1 : c;
    return r * ncols + c;
}

ELFI_HD bool sa_get(const uint32_t* lat, int s) { return (lat[s >> 5] >> (s & 31)) & 1u; }

// The law on one row, sequentially: lat (sa_words(N) words) holds the initial lattice and ends as
// the last frame's; list has room for N entries.  frame(k, lat) is called for k = 0 .. num_obs with
// the lattice of frame k.  Used by the host build; the kernel runs the same steps warp-wide.
template <class Frame>
ELFI_HD void sa_simulate_row(const Philox& ph, uint64_t row, double pm, double pp, uint32_t* lat,
                             uint16_t* list, int nrows, int ncols, int num_obs, int interval,
                             Frame&& frame) {
    const int N = nrows * ncols, W = sa_words(N);
    frame(0, lat);
    const int iters = num_obs * interval;
    for (int t = 0; t < iters; ++t) {
        int n = 0;
        for (int w = 0; w < W; ++w)
            for (uint32_t bits = lat[w]; bits; bits &= bits - 1)
                list[n++] = uint16_t(w * 32 + sa_ctz(bits));
        if (n < N) {
            for (int s = 0; pm > 0 && s < n; ++s) {
                const SaSlot sl = sa_slot(ph, row, t, 0, s, n, pm);
                if (!sl.kept) continue;
                const int from = list[sl.index], to = sa_target(from, sl.dir, nrows, ncols);
                if (!sa_get(lat, to)) {
                    lat[from >> 5] &= ~(1u << (from & 31));
                    lat[to >> 5] |= 1u << (to & 31);
                    list[sl.index] = uint16_t(to);
                }
            }
            for (int s = 0; pp > 0 && s < n; ++s) {
                const SaSlot sl = sa_slot(ph, row, t, 1, s, n, pp);
                if (!sl.kept) continue;
                const int to = sa_target(list[sl.index], sl.dir, nrows, ncols);
                lat[to >> 5] |= 1u << (to & 31);
            }
        }
        if ((t + 1) % interval == 0) frame((t + 1) / interval, lat);
    }
}

}  // namespace elfi
