// common.cuh -- shared plumbing for the elfi_b200 CUDA library (sm_90a only).
//
// Error model of the C ABI: every entry point returns 0 on success and a negative
// code on failure; the message is kept per host thread and read back with
// elfi_b200_last_error().  No exceptions cross the ABI.
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <type_traits>

#include "../../include/elfi_b200.h"

namespace elfi {

void set_error(const char* fmt, ...);

#define ELFI_CUDA_OK(expr)                                                              \
    do {                                                                                \
        cudaError_t _e = (expr);                                                        \
        if (_e != cudaSuccess) {                                                        \
            ::elfi::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),   \
                              __FILE__, __LINE__);                                      \
            cudaGetLastError(); /* clear the (non-sticky) error for later calls */      \
            return ELFI_B200_ERR_CUDA;                                                  \
        }                                                                               \
    } while (0)

#define ELFI_REQUIRE(cond, ...)                                                         \
    do {                                                                                \
        if (!(cond)) {                                                                  \
            ::elfi::set_error(__VA_ARGS__);                                             \
            return ELFI_B200_ERR_ARG;                                                   \
        }                                                                               \
    } while (0)

typedef CUresult (*tensor_map_encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                         const cuuint64_t*, const cuuint64_t*,
                                         const cuuint32_t*, const cuuint32_t*,
                                         CUtensorMapInterleave, CUtensorMapSwizzle,
                                         CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

}  // namespace elfi

// Opaque per-device context: device properties, the driver entry point used to encode
// TMA descriptors, and a grow-only scratch arena (mask words, radix-sort ping-pong
// buffers, partial reductions) so the hot calls never allocate.
struct elfi_b200_ctx {
    int device;
    int sm_count;
    size_t smem_optin;
    elfi::tensor_map_encode_fn encode_tiled;
    void* scratch;
    size_t scratch_bytes;
    // the GP Cholesky look-ahead's second stream and its two ordering events (gp.cu)
    cudaStream_t side_stream;
    cudaEvent_t side_event[2];
};

namespace elfi {

// Returns a device pointer to at least `bytes` of scratch (256-byte aligned), or nullptr
// after set_error().  Growth synchronises the device: it only happens on the first calls.
void* ctx_scratch(elfi_b200_ctx* ctx, size_t bytes);

// Encodes a rank-2 fp64 tensor map over a row-major (rows, cols) matrix with leading
// dimension `ld` (elements) and a (box_rows x 16) box, 128-byte swizzle.
int make_rowmajor_f64_map(elfi_b200_ctx* ctx, const double* base, int64_t rows, int64_t cols,
                          int64_t ld, int box_rows, CUtensorMap* out);

inline bool tma_compatible(const void* base, int64_t ld) {
    return (reinterpret_cast<uintptr_t>(base) % 16 == 0) && ((ld * 8) % 16 == 0);
}

// The body of a device entry point, after its argument checks: make the context's device current,
// run body(stream), which returns ELFI_B200_OK or an error code (so ELFI_CUDA_OK and ELFI_REQUIRE
// work inside it), then report an error of the launches it made.
template <class Body>
int run_on_device(elfi_b200_ctx* ctx, void* stream, Body&& body) {
    ELFI_CUDA_OK(cudaSetDevice(ctx->device));
    const int rc = body(static_cast<cudaStream_t>(stream));
    if (rc != ELFI_B200_OK) return rc;
    ELFI_CUDA_OK(cudaGetLastError());
    return ELFI_B200_OK;
}

// f(std::integral_constant<int, K>{}) for the power of two K in [LO, HI] that k selects (LO below
// the range, HI above it); instantiates f for exactly LO, 2 LO, ..., HI.  Returns what f returns.
template <int LO, int HI, class F>
auto with_pow2(int k, F&& f) {
    if constexpr (LO == HI) {
        return f(std::integral_constant<int, LO>{});
    } else {
        if (k <= LO) return f(std::integral_constant<int, LO>{});
        return with_pow2<2 * LO, HI>(k, f);
    }
}

// ceil(work / per_block) blocks, at most ctas_per_sm per SM: the kernels behind it grid-stride
inline unsigned capped_grid(const elfi_b200_ctx* ctx, int64_t work, int64_t per_block,
                            int ctas_per_sm) {
    const int64_t blocks = (work + per_block - 1) / per_block;
    const int64_t cap = int64_t(ctx->sm_count) * ctas_per_sm;
    return unsigned(blocks < cap ? blocks : cap);
}

// ------------------------------------------------------------------------------------
// Device-side PTX helpers (mbarrier + TMA).  All addresses are shared::cta 32-bit.
// ------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}

__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
                 : "memory");
}

__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}

__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}

// 2-D tiled TMA load: box at (col0, row0) of the tensor map -> shared memory, completion
// signalled on `bar` with the box byte count.
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int32_t col0,
                                            int32_t row0, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%2, %3}], [%4];"
        ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(col0), "r"(row0), "r"(bar)
        : "memory");
}

// 1-D bulk copy global -> shared (`bytes` a multiple of 16, both addresses 16-byte aligned),
// completion signalled on `bar` with the byte count.
__device__ __forceinline__ void bulk_load_1d(uint32_t dst, const void* src, uint32_t bytes,
                                             uint32_t bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
        ::"r"(dst), "l"(src), "r"(bytes), "r"(bar)
        : "memory");
}

__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

}  // namespace elfi
