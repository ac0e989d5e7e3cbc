// ctx.cu -- context, error string, scratch arena and TMA descriptor encoding.
#include "common.cuh"

namespace elfi {

static thread_local char g_error[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_error, sizeof(g_error), fmt, ap);
    va_end(ap);
}

void* ctx_scratch(elfi_b200_ctx* ctx, size_t bytes) {
    if (bytes <= ctx->scratch_bytes) return ctx->scratch;
    size_t want = bytes + (bytes >> 2) + (1u << 20);
    want = (want + 255) & ~size_t(255);
    if (ctx->scratch) {
        if (cudaDeviceSynchronize() != cudaSuccess || cudaFree(ctx->scratch) != cudaSuccess) {
            set_error("scratch release failed: %s", cudaGetErrorString(cudaGetLastError()));
            ctx->scratch = nullptr;
            ctx->scratch_bytes = 0;
            return nullptr;
        }
        ctx->scratch = nullptr;
        ctx->scratch_bytes = 0;
    }
    void* p = nullptr;
    cudaError_t e = cudaMalloc(&p, want);
    if (e != cudaSuccess) {
        set_error("cudaMalloc(%zu) for scratch failed: %s", want, cudaGetErrorString(e));
        cudaGetLastError();
        return nullptr;
    }
    ctx->scratch = p;
    ctx->scratch_bytes = want;
    return p;
}

int make_rowmajor_f64_map(elfi_b200_ctx* ctx, const double* base, int64_t rows, int64_t cols,
                          int64_t ld, int box_rows, CUtensorMap* out) {
    ELFI_REQUIRE(ctx->encode_tiled != nullptr, "cuTensorMapEncodeTiled entry point unavailable");
    ELFI_REQUIRE(tma_compatible(base, ld), "matrix is not TMA compatible (16-byte base/stride)");
    cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
    cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld) * sizeof(double)};
    cuuint32_t box[2] = {16u, static_cast<cuuint32_t>(box_rows)};
    cuuint32_t estr[2] = {1u, 1u};
    CUresult r = ctx->encode_tiled(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 2,
                                   const_cast<double*>(base), dims, strides, box, estr,
                                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed with CUresult %d (rows=%lld cols=%lld ld=%lld)",
                  static_cast<int>(r), (long long)rows, (long long)cols, (long long)ld);
        return ELFI_B200_ERR_CUDA;
    }
    return ELFI_B200_OK;
}

}  // namespace elfi

extern "C" {

int elfi_b200_version(void) { return ELFI_B200_VERSION; }

const char* elfi_b200_last_error(void) { return elfi::g_error; }

int elfi_b200_ctx_create(int device, elfi_b200_ctx** out) {
    ELFI_REQUIRE(out != nullptr, "ctx_create: out is NULL");
    *out = nullptr;
    int count = 0;
    ELFI_CUDA_OK(cudaGetDeviceCount(&count));
    ELFI_REQUIRE(device >= 0 && device < count, "ctx_create: device %d out of range (%d visible)",
                 device, count);
    ELFI_CUDA_OK(cudaSetDevice(device));
    cudaDeviceProp prop;
    ELFI_CUDA_OK(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {
        elfi::set_error("ctx_create: device %d is sm_%d%d; this library is built for sm_90a only",
                        device, prop.major, prop.minor);
        return ELFI_B200_ERR_UNSUPPORTED;
    }
    elfi_b200_ctx* ctx = new elfi_b200_ctx();
    memset(ctx, 0, sizeof(*ctx));
    ctx->device = device;
    ctx->sm_count = prop.multiProcessorCount;
    ctx->smem_optin = prop.sharedMemPerBlockOptin;
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || fn == nullptr) {
        elfi::set_error("ctx_create: cuTensorMapEncodeTiled not available from the driver");
        delete ctx;
        cudaGetLastError();
        return ELFI_B200_ERR_CUDA;
    }
    ctx->encode_tiled = reinterpret_cast<elfi::tensor_map_encode_fn>(fn);
    for (int i = 0; i < 2; ++i)
        ELFI_CUDA_OK(cudaStreamCreateWithFlags(&ctx->copy_stream[i], cudaStreamNonBlocking));
    for (int i = 0; i < 4; ++i)
        ELFI_CUDA_OK(cudaEventCreateWithFlags(&ctx->copy_event[i], cudaEventDisableTiming));
    *out = ctx;
    return ELFI_B200_OK;
}

int elfi_b200_ctx_destroy(elfi_b200_ctx* ctx) {
    if (!ctx) return ELFI_B200_OK;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    if (ctx->scratch) cudaFree(ctx->scratch);
    if (ctx->dev_stage) cudaFree(ctx->dev_stage);
    if (ctx->pinned) cudaFreeHost(ctx->pinned);
    for (int i = 0; i < 2; ++i)
        if (ctx->copy_stream[i]) cudaStreamDestroy(ctx->copy_stream[i]);
    for (int i = 0; i < 4; ++i)
        if (ctx->copy_event[i]) cudaEventDestroy(ctx->copy_event[i]);
    delete ctx;
    return ELFI_B200_OK;
}

int elfi_b200_ctx_sm_count(const elfi_b200_ctx* ctx) { return ctx ? ctx->sm_count : 0; }

// Single-process multi-GPU exchange of accepted particles (SURVEY.md section 8b/8e): one context
// per GPU; GPU g contributes send[g] (rows x width doubles in its memory) and receives the
// context-ordered concatenation in recv[g].  Peer copies (cudaMemcpyPeerAsync, NVLink when peer
// access can be enabled) ordered by events: a destination stream waits until every source has
// produced its block; every source stream waits until all destinations have read it, so the
// caller may overwrite send[g] with later work on streams[g].
int elfi_b200_allgather_particles(elfi_b200_ctx* const* ctxs, int64_t n_ctx, const double* const* send,
                                  int64_t rows, int64_t width, double* const* recv,
                                  void* const* streams) {
    ELFI_REQUIRE(ctxs && send && recv && streams && n_ctx >= 1 && n_ctx <= 64,
                 "allgather_particles: bad argument");
    ELFI_REQUIRE(rows >= 0 && width >= 1, "allgather_particles: bad shape");
    for (int64_t g = 0; g < n_ctx; ++g)
        ELFI_REQUIRE(ctxs[g] && (rows == 0 || (send[g] && recv[g])), "allgather_particles: NULL entry %lld",
                     (long long)g);
    if (rows == 0) return ELFI_B200_OK;
    const size_t bytes = size_t(rows) * size_t(width) * 8;
    int caller_device = 0;
    ELFI_CUDA_OK(cudaGetDevice(&caller_device));
    struct Restore {
        int d;
        ~Restore() { cudaSetDevice(d); }
    } restore{caller_device};   // the calling thread keeps its current device
    // peer access (once per ordered pair; "already enabled" is not an error)
    for (int64_t d = 0; d < n_ctx; ++d) {
        ELFI_CUDA_OK(cudaSetDevice(ctxs[d]->device));
        for (int64_t s = 0; s < n_ctx; ++s) {
            if (ctxs[s]->device == ctxs[d]->device) continue;
            int can = 0;
            ELFI_CUDA_OK(cudaDeviceCanAccessPeer(&can, ctxs[d]->device, ctxs[s]->device));
            if (can) {
                cudaError_t e = cudaDeviceEnablePeerAccess(ctxs[s]->device, 0);
                if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) ELFI_CUDA_OK(e);
                cudaGetLastError();
            }
        }
    }
    // ready[g]: send[g] is complete on its stream
    for (int64_t g = 0; g < n_ctx; ++g) {
        ELFI_CUDA_OK(cudaSetDevice(ctxs[g]->device));
        ELFI_CUDA_OK(cudaEventRecord(ctxs[g]->copy_event[2], static_cast<cudaStream_t>(streams[g])));
    }
    for (int64_t d = 0; d < n_ctx; ++d) {
        ELFI_CUDA_OK(cudaSetDevice(ctxs[d]->device));
        cudaStream_t sd = static_cast<cudaStream_t>(streams[d]);
        for (int64_t s = 0; s < n_ctx; ++s) {
            if (s != d) ELFI_CUDA_OK(cudaStreamWaitEvent(sd, ctxs[s]->copy_event[2], 0));
            ELFI_CUDA_OK(cudaMemcpyPeerAsync(recv[d] + size_t(s) * rows * width, ctxs[d]->device, send[s],
                                             ctxs[s]->device, bytes, sd));
        }
        ELFI_CUDA_OK(cudaEventRecord(ctxs[d]->copy_event[3], sd));   // done[d]: d has read every block
    }
    for (int64_t s = 0; s < n_ctx; ++s) {
        ELFI_CUDA_OK(cudaSetDevice(ctxs[s]->device));
        for (int64_t d = 0; d < n_ctx; ++d)
            if (d != s)
                ELFI_CUDA_OK(cudaStreamWaitEvent(static_cast<cudaStream_t>(streams[s]),
                                                 ctxs[d]->copy_event[3], 0));
    }
    return ELFI_B200_OK;
}

}  // extern "C"
