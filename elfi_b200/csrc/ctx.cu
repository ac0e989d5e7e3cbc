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
    ELFI_CUDA_OK(cudaStreamCreateWithFlags(&ctx->side_stream, cudaStreamNonBlocking));
    for (int i = 0; i < 2; ++i)
        ELFI_CUDA_OK(cudaEventCreateWithFlags(&ctx->side_event[i], cudaEventDisableTiming));
    *out = ctx;
    return ELFI_B200_OK;
}

int elfi_b200_ctx_destroy(elfi_b200_ctx* ctx) {
    if (!ctx) return ELFI_B200_OK;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    elfi::usersim_free_all(ctx);
    if (ctx->scratch) cudaFree(ctx->scratch);
    if (ctx->side_stream) cudaStreamDestroy(ctx->side_stream);
    for (int i = 0; i < 2; ++i)
        if (ctx->side_event[i]) cudaEventDestroy(ctx->side_event[i]);
    delete ctx;
    return ELFI_B200_OK;
}

int elfi_b200_ctx_sm_count(const elfi_b200_ctx* ctx) { return ctx ? ctx->sm_count : 0; }

}  // extern "C"
