// rowstream.cuh -- the streaming skeleton shared by every "one result per row" kernel on the
// sampler hot path (Euclidean / nested distances, MA2 autocovariance, mean/variance).
//
// Why this shape.  The reference's arithmetic is *sequential along a row* (SciPy's cdist sums
// j = 0..D-1 left to right; NumPy's pairwise sum has a fixed tree), and results must be
// bit-identical, so a row cannot be split across lanes.  One lane therefore owns one row and
// walks it in order.  Read straight from global memory that is a 32-way uncoalesced access
// (lanes are ld*8 bytes apart), so the (B, D) matrix is staged through shared memory by TMA:
//
//   * a rank-2 tensor map over the row-major matrix, box = 32 rows x 16 fp64 columns
//     (32 x 128 B = 4 KiB), SWIZZLE_128B;
//   * with the 128-byte swizzle the 16-byte chunk c of row r lands at
//     r*128 + ((c ^ (r & 7)) << 4), so the eight lanes of a quarter-warp reading chunk c of
//     eight consecutive rows hit eight distinct 16-byte bank groups: LDS.128 without bank
//     conflicts, no padding, no manual transpose;
//   * every warp is its own producer and consumer: it owns NS box slots and NS mbarriers,
//     lane 0 re-arms a slot and issues the next TMA right after the warp has consumed it
//     (__syncwarp orders the reads before the async-proxy overwrite).  No block-level
//     barrier, no dedicated producer warp, no empty-barrier round trip;
//   * boxes are consumed in (row tile, column group) order, column groups of one tile back
//     to back, so a lane sees its row strictly left to right;
//   * out-of-range rows / columns are zero-filled by TMA and always deliver the full box
//     byte count, so the expect_tx value is a constant 4096.
//
// Bytes in flight per SM = WARPS * (NS-1) * 4 KiB (160 KiB at WARPS=8, NS=6): several times
// the ~25 KiB per SM that Little's law asks for 3.35 TB/s (H100 SXM data sheet) at ~1 us of
// latency over 132 SMs, so HBM latency is covered
// without relying on occupancy.  Grid = one persistent CTA per SM; tiles are dealt
// round-robin to the global warp index.
#pragma once

#include <type_traits>

#include "common.cuh"

namespace elfi {

// Optional parts of the Consumer concept, detected at compile time:
//   static constexpr bool RS_TILE_INFO = true;   void set_tile(int64_t row0, int64_t B);
//       -- told the first row of every tile before its first box (e.g. to mask rows >= B when a
//          consumer also reduces DOWN the rows of a box)
//   static constexpr bool RS_FINISH = true;      void finish(int64_t gw, int lane);
//       -- called once per warp after its last box (flush per-warp accumulators)
template <class C, class = void> struct rs_has_tile_info : std::false_type {};
template <class C> struct rs_has_tile_info<C, std::void_t<decltype(C::RS_TILE_INFO)>> : std::true_type {};
template <class C, class = void> struct rs_has_finish : std::false_type {};
template <class C> struct rs_has_finish<C, std::void_t<decltype(C::RS_FINISH)>> : std::true_type {};

constexpr int RS_WARPS = 8;          // consumer warps per CTA (default; see WARPS below)
constexpr int RS_BOX_ROWS = 32;      // rows per box (one per lane)
constexpr int RS_BOX_COLS = 16;      // fp64 columns per box (128 bytes)
constexpr int RS_BOX_BYTES = RS_BOX_ROWS * RS_BOX_COLS * 8;
constexpr int RS_MAX_STAGES = 6;

// D rounded up to whole boxes: the row length of everything a consumer keeps per column in
// shared memory (TMA zero-fills the columns >= D of the last box).
template <class Int>
__host__ __device__ constexpr Int rs_padded_cols(Int D) {
    return ((D + RS_BOX_COLS - 1) / RS_BOX_COLS) * RS_BOX_COLS;
}

// Shared-memory layout (dynamic, 1024-byte aligned):
//   [RS_WARPS][ns][4096]  boxes
//   [RS_WARPS][ns] u64    mbarriers
//   consumer area         (obs / weights ...), 16-byte aligned
__host__ __device__ inline size_t rs_box_bytes(int ns, int warps = RS_WARPS) {
    return size_t(warps) * ns * RS_BOX_BYTES;
}
__host__ __device__ inline size_t rs_bar_bytes(int ns, int warps = RS_WARPS) {
    return size_t(warps) * ns * 8;
}
__host__ __device__ inline size_t rs_aux_offset(int ns, int warps = RS_WARPS) {
    return (rs_box_bytes(ns, warps) + rs_bar_bytes(ns, warps) + 15) & ~size_t(15);
}

// Picks the deepest pipeline that fits next to `aux_bytes` of consumer shared memory.
inline int rs_pick_stages(size_t smem_optin, size_t aux_bytes, int warps = RS_WARPS) {
    for (int ns = RS_MAX_STAGES; ns >= 2; --ns)
        if (rs_aux_offset(ns, warps) + aux_bytes + 1024 <= smem_optin) return ns;
    return 0;
}

// Does the (.., D) matrix M take the row stream with `aux_bytes` of consumer shared memory?  It
// needs one whole box of columns, a TMA-addressable base and stride, and room for a 2-slot ring;
// callers send every other matrix to their thread-per-row kernel.
inline bool rs_streams(const elfi_b200_ctx* ctx, const void* M, int64_t ld, int64_t D,
                       size_t aux_bytes) {
    return D >= RS_BOX_COLS && tma_compatible(M, ld) &&
           rs_pick_stages(ctx->smem_optin, aux_bytes) >= 2;
}

// The Consumer concept (all members are per lane):
//   struct Params;                                    // POD passed by value to the kernel
//   static void setup_shared(uint8_t* aux, const Params&, int D);   // CTA-cooperative
//   Consumer(const Params&, const uint8_t* aux, int D, int lane);
//   static constexpr int PASSES;                      // times a tile's boxes are streamed
//   void begin_row();
//   void consume(int pass, int cg, const uint8_t* box_row, int sw);  // 16 columns of my row
//   void end_row(int64_t row, int64_t B, int lane);   // row may be >= B (zero-filled tile)
// With PASSES > 1 a tile's column groups are requested again right after the first sweep
// (second sweep hits L2: a tile is at most a few tens of KiB), e.g. mean then variance.
//
// WARPS: consumers whose per-element arithmetic is a long dependent fp64 chain (nested distances,
// fused column moments) cannot hide its latency with two warps per scheduler; they may run with
// 12 warps and a shallower ring (the bytes in flight, WARPS * (ns-1) * 4 KiB, stay above the
// Little's-law requirement).  A consumer sees the count as blockDim.x >> 5.
template <class Consumer, int WARPS = RS_WARPS>
__global__ void __launch_bounds__(WARPS * 32, 1)
rowstream_kernel(const __grid_constant__ CUtensorMap map, int64_t B, int D, int ns,
                 typename Consumer::Params params) {
    extern __shared__ __align__(1024) uint8_t smem[];
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    uint8_t* aux = smem + rs_aux_offset(ns, WARPS);

    Consumer::setup_shared(aux, params, D);

    const uint32_t box0 = smem_u32(smem) + uint32_t(warp) * ns * RS_BOX_BYTES;
    const uint32_t bar0 = smem_u32(smem + rs_box_bytes(ns, WARPS)) + uint32_t(warp) * ns * 8;
    const uint8_t* box0_generic = smem + size_t(warp) * ns * RS_BOX_BYTES;

    if (lane == 0) {
        if (warp == 0) tma_prefetch_desc(&map);
        for (int s = 0; s < ns; ++s) mbar_init(bar0 + s * 8, 1);
        mbar_fence_init();
    }
    __syncthreads();  // setup_shared visible; barriers initialised

    const int Gc = (D + RS_BOX_COLS - 1) / RS_BOX_COLS;   // column groups per sweep
    const int G = Gc * Consumer::PASSES;                  // boxes per tile
    const int64_t ntiles = (B + RS_BOX_ROWS - 1) / RS_BOX_ROWS;
    const int64_t gw = int64_t(blockIdx.x) * WARPS + warp;
    const int64_t GW = int64_t(gridDim.x) * WARPS;
    const int64_t my_tiles = gw < ntiles ? (ntiles - gw + GW - 1) / GW : 0;
    const int64_t nbox = my_tiles * G;

    // producer cursor (lane 0 only): next box to request
    int64_t p_tile = gw;
    int p_cg = 0;
    int p_col = 0;
    int64_t p_q = 0;
    int p_s = 0;
    auto issue = [&]() {
        mbar_arrive_expect_tx(bar0 + p_s * 8, RS_BOX_BYTES);
        tma_load_2d(box0 + p_s * RS_BOX_BYTES, &map, p_col * RS_BOX_COLS,
                    int32_t(p_tile * RS_BOX_ROWS), bar0 + p_s * 8);
        ++p_q;
        if (++p_s == ns) p_s = 0;
        if (++p_col == Gc) p_col = 0;
        if (++p_cg == G) { p_cg = 0; p_tile += GW; }
    };
    if (lane == 0) {
        const int64_t pre = nbox < ns ? nbox : ns;
        for (int64_t i = 0; i < pre; ++i) issue();
    }

    Consumer c(params, aux, D, lane);
    const int sw = lane & 7;
    const uint32_t row_off = uint32_t(lane) * 128;

    int s = 0;
    uint32_t parity = 0;
    int cg = 0;
    int col = 0;
    int pass = 0;
    int64_t tile = gw;
    for (int64_t q = 0; q < nbox; ++q) {
        mbar_wait(bar0 + s * 8, parity);
        if (cg == 0) {
            c.begin_row();
            if constexpr (rs_has_tile_info<Consumer>::value) c.set_tile(tile * RS_BOX_ROWS, B);
        }
        c.consume(pass, col, box0_generic + size_t(s) * RS_BOX_BYTES + row_off, sw);
        __syncwarp();
        if (lane == 0 && p_q < nbox) issue();
        if (cg == G - 1) c.end_row(tile * RS_BOX_ROWS + lane, B, lane);
        if (++col == Gc) { col = 0; ++pass; }
        if (++cg == G) { cg = 0; pass = 0; tile += GW; }
        if (++s == ns) { s = 0; parity ^= 1; }
    }
    if constexpr (rs_has_finish<Consumer>::value) {
        __syncwarp();
        c.finish(gw, lane);
    }
}

// Host-side launcher: encodes the tensor map, sizes the pipeline and the persistent grid.
template <class Consumer, int WARPS = RS_WARPS>
int rowstream_launch(elfi_b200_ctx* ctx, const double* M, int64_t ld, int64_t B, int64_t D,
                     size_t aux_bytes, const typename Consumer::Params& params,
                     cudaStream_t stream) {
    ELFI_REQUIRE(D <= (int64_t(1) << 30) && B < (int64_t(1) << 31),
                 "matrix too large for int32 TMA coordinates (B=%lld, D=%lld)", (long long)B,
                 (long long)D);
    if (B == 0) return ELFI_B200_OK;
    const int ns = rs_pick_stages(ctx->smem_optin, aux_bytes, WARPS);
    ELFI_REQUIRE(ns >= 2, "row too wide for the shared-memory pipeline (D=%lld)", (long long)D);
    CUtensorMap map;
    int rc = make_rowmajor_f64_map(ctx, M, B, D, ld, RS_BOX_ROWS, &map);
    if (rc) return rc;
    const size_t smem_bytes = rs_aux_offset(ns, WARPS) + aux_bytes;
    auto kern = rowstream_kernel<Consumer, WARPS>;
    ELFI_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      int(smem_bytes)));
    const int64_t ntiles = (B + RS_BOX_ROWS - 1) / RS_BOX_ROWS;
    int64_t ctas = (ntiles + WARPS - 1) / WARPS;
    if (ctas > ctx->sm_count) ctas = ctx->sm_count;
    kern<<<dim3(unsigned(ctas)), dim3(WARPS * 32), smem_bytes, stream>>>(map, B, int(D), ns, params);
    ELFI_CUDA_OK(cudaGetLastError());
    return ELFI_B200_OK;
}

}  // namespace elfi
