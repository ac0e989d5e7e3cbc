// usersim.cu -- user-written simulators in throughput mode: NVRTC compiles the user's per-row
// device functions together with the harness kernel of usersim_rt.cuh for sm_90a, the runtime
// loads the CUBIN (cudaLibraryLoadData, no driver API link), and the context keeps the result
// under (source, p, n_out, n_sum, salt) so that a model rebuilt with the same source compiles
// once.  The contract the source follows is in usersim_rt.cuh and include/elfi_b200.h.
#include <dlfcn.h>
#include <nvrtc.h>

#include <string>
#include <vector>

#include "common.cuh"

// One compiled simulator: a kernel per mode (nullptr where the shapes rule the mode out).
struct elfi_b200_usersim {
    std::string source;
    int p, n_out, n_sum;
    uint32_t salt;
    int refs;
    cudaLibrary_t library;
    cudaKernel_t kernel[4];
    elfi_b200_usersim* next;
};

namespace elfi {

namespace {

constexpr int kUsersimModes = 4;
constexpr int kUsersimBlock = 128;   // usersim_kernel's __launch_bounds__

// csrc/ beside the directory of this library (lib/libelfi_b200.so): where usersim_rt.cuh and the
// headers it includes live
std::string csrc_dir() {
    Dl_info info;
    if (dladdr(reinterpret_cast<void*>(&elfi_b200_usersim_compile), &info) == 0 ||
        info.dli_fname == nullptr)
        return std::string();
    std::string path(info.dli_fname);
    const size_t slash = path.rfind('/');
    std::string lib_dir = slash == std::string::npos ? std::string(".") : path.substr(0, slash);
    return lib_dir + "/../csrc";
}

bool mode_available(int mode, int n_out, int n_sum) {
    if (mode == 0) return true;
    if (n_sum == 0) return false;
    return mode != 2 || n_out <= ELFI_B200_USERSIM_LOCAL_MAX;
}

void copy_log(char* log, int64_t log_len, const std::string& text) {
    if (log == nullptr || log_len <= 0) return;
    const size_t n = text.size() < size_t(log_len - 1) ? text.size() : size_t(log_len - 1);
    memcpy(log, text.data(), n);
    log[n] = '\0';
}

// NVRTC -> CUBIN -> library and kernels of `sim`; returns ELFI_B200_OK or an error (log filled)
int usersim_build(elfi_b200_usersim* sim, char* log, int64_t log_len) {
    const std::string dir = csrc_dir();
    ELFI_REQUIRE(!dir.empty(), "usersim_compile: cannot locate the library's csrc directory");
    // #line: the NVRTC log numbers the user's lines as the user wrote them
    const std::string text = "#include \"usersim_rt.cuh\"\n#line 1 \"user_source\"\n" + sim->source +
                             "\n";
    nvrtcProgram prog;
    nvrtcResult r = nvrtcCreateProgram(&prog, text.c_str(), "usersim.cu", 0, nullptr, nullptr);
    if (r != NVRTC_SUCCESS) {
        set_error("usersim_compile: nvrtcCreateProgram failed: %s", nvrtcGetErrorString(r));
        return ELFI_B200_ERR_UNSUPPORTED;
    }
    std::string names[kUsersimModes];
    for (int m = 0; m < kUsersimModes; ++m) {
        if (!mode_available(m, sim->n_out, sim->n_sum)) continue;
        names[m] = "elfi::usersim_kernel<" + std::to_string(sim->p) + ", " +
                   std::to_string(sim->n_out) + ", " + std::to_string(sim->n_sum) + ", " +
                   std::to_string(m) + ">";
        nvrtcAddNameExpression(prog, names[m].c_str());
    }
    char defs[4][64];
    snprintf(defs[0], sizeof(defs[0]), "-DELFI_B200_USERSIM_SALT=0x%08xu", sim->salt);
    snprintf(defs[1], sizeof(defs[1]), "-DELFI_B200_USERSIM_P=%d", sim->p);
    snprintf(defs[2], sizeof(defs[2]), "-DELFI_B200_USERSIM_N_OUT=%d", sim->n_out);
    snprintf(defs[3], sizeof(defs[3]), "-DELFI_B200_USERSIM_N_SUM=%d", sim->n_sum);
    const std::string include = "-I" + dir;
    const char* opts[] = {"--gpu-architecture=sm_90a", "-std=c++17", include.c_str(), defs[0],
                          defs[1], defs[2], defs[3]};
    r = nvrtcCompileProgram(prog, 7, opts);
    if (r != NVRTC_SUCCESS) {
        size_t n = 0;
        nvrtcGetProgramLogSize(prog, &n);
        std::string plog(n, '\0');
        if (n) nvrtcGetProgramLog(prog, &plog[0]);
        while (!plog.empty() && plog.back() == '\0') plog.pop_back();
        copy_log(log, log_len, plog);
        nvrtcDestroyProgram(&prog);
        set_error("usersim_compile: NVRTC could not compile the simulator (%s); its log: %.300s",
                  nvrtcGetErrorString(r), plog.c_str());
        return ELFI_B200_ERR_ARG;
    }
    size_t cubin_size = 0;
    nvrtcGetCUBINSize(prog, &cubin_size);
    std::vector<char> cubin(cubin_size);
    nvrtcGetCUBIN(prog, cubin.data());
    std::string lowered[kUsersimModes];
    for (int m = 0; m < kUsersimModes; ++m) {
        const char* name = nullptr;
        if (!names[m].empty() && nvrtcGetLoweredName(prog, names[m].c_str(), &name) == NVRTC_SUCCESS)
            lowered[m] = name;
    }
    nvrtcDestroyProgram(&prog);
    ELFI_CUDA_OK(cudaLibraryLoadData(&sim->library, cubin.data(), nullptr, nullptr, 0, nullptr,
                                     nullptr, 0));
    for (int m = 0; m < kUsersimModes; ++m) {
        sim->kernel[m] = nullptr;
        if (names[m].empty()) continue;
        cudaError_t e = lowered[m].empty() ? cudaErrorSymbolNotFound
                                           : cudaLibraryGetKernel(&sim->kernel[m], sim->library,
                                                                  lowered[m].c_str());
        if (e != cudaSuccess) {
            set_error("usersim_compile: kernel %s not found in the compiled library: %s",
                      names[m].c_str(), cudaGetErrorString(e));
            cudaGetLastError();
            cudaLibraryUnload(sim->library);
            return ELFI_B200_ERR_CUDA;
        }
    }
    return ELFI_B200_OK;
}

void usersim_free(elfi_b200_usersim* sim) {
    cudaLibraryUnload(sim->library);
    delete sim;
}

}  // namespace

void usersim_free_all(elfi_b200_ctx* ctx) {
    while (ctx->usersims) {
        elfi_b200_usersim* next = ctx->usersims->next;
        usersim_free(ctx->usersims);
        ctx->usersims = next;
    }
}

}  // namespace elfi

extern "C" {

int elfi_b200_usersim_compile(elfi_b200_ctx* ctx, const char* source, int64_t p, int64_t n_out,
                              int64_t n_sum, uint64_t salt, char* log, int64_t log_len,
                              elfi_b200_usersim** handle) {
    ELFI_REQUIRE(ctx != nullptr && source != nullptr && handle != nullptr,
                 "usersim_compile: ctx, source and handle must not be NULL");
    *handle = nullptr;
    elfi::copy_log(log, log_len, "");
    ELFI_REQUIRE(p >= 1 && p <= ELFI_B200_USERSIM_P_MAX,
                 "usersim_compile: 1 <= p <= %d parameters, got %lld", ELFI_B200_USERSIM_P_MAX,
                 (long long)p);
    ELFI_REQUIRE(n_out >= 1 && n_out <= ELFI_B200_USERSIM_N_OUT_MAX,
                 "usersim_compile: 1 <= n_out <= %d, got %lld", ELFI_B200_USERSIM_N_OUT_MAX,
                 (long long)n_out);
    ELFI_REQUIRE(n_sum >= 0 && n_sum <= ELFI_B200_USERSIM_N_SUM_MAX,
                 "usersim_compile: 0 <= n_sum <= %d, got %lld", ELFI_B200_USERSIM_N_SUM_MAX,
                 (long long)n_sum);
    ELFI_REQUIRE(salt <= 0xffffffffull, "usersim_compile: the salt is a 32-bit word, got %llu",
                 (unsigned long long)salt);
    for (elfi_b200_usersim* s = ctx->usersims; s; s = s->next) {
        if (s->p == p && s->n_out == n_out && s->n_sum == n_sum && s->salt == salt &&
            s->source == source) {
            ++s->refs;
            *handle = s;
            return ELFI_B200_OK;
        }
    }
    ELFI_CUDA_OK(cudaSetDevice(ctx->device));
    elfi_b200_usersim* sim = new elfi_b200_usersim();
    sim->source = source;
    sim->p = int(p);
    sim->n_out = int(n_out);
    sim->n_sum = int(n_sum);
    sim->salt = uint32_t(salt);
    sim->refs = 1;
    const int rc = elfi::usersim_build(sim, log, log_len);
    if (rc != ELFI_B200_OK) {
        delete sim;
        return rc;
    }
    sim->next = ctx->usersims;
    ctx->usersims = sim;
    *handle = sim;
    return ELFI_B200_OK;
}

int elfi_b200_usersim_launch(elfi_b200_ctx* ctx, const elfi_b200_usersim* handle,
                             const double* const* theta_cols_host, int64_t B, uint64_t key,
                             uint64_t offset, int32_t mode, double* Y, int64_t ldY, double* S,
                             int64_t ldS, void* stream) {
    ELFI_REQUIRE(ctx != nullptr && handle != nullptr, "usersim_launch: ctx and handle must not be NULL");
    ELFI_REQUIRE(mode >= 0 && mode < elfi::kUsersimModes, "usersim_launch: mode %d is not 0-3",
                 int(mode));
    ELFI_REQUIRE(handle->kernel[mode] != nullptr,
                 "usersim_launch: mode %d needs n_sum > 0%s (n_out = %d, n_sum = %d)", int(mode),
                 mode == 2 ? " and n_out <= ELFI_B200_USERSIM_LOCAL_MAX" : "", handle->n_out,
                 handle->n_sum);
    ELFI_REQUIRE(B >= 0 && (B + elfi::kUsersimBlock - 1) / elfi::kUsersimBlock <= 0x7fffffff,
                 "usersim_launch: batch size %lld out of range", (long long)B);
    const bool data = mode != 2, summaries = mode != 0, simulates = mode != 3;
    ELFI_REQUIRE(!data || (Y != nullptr && ldY >= handle->n_out),
                 "usersim_launch: mode %d needs Y with ldY >= n_out = %d", int(mode), handle->n_out);
    ELFI_REQUIRE(!summaries || (S != nullptr && ldS >= handle->n_sum),
                 "usersim_launch: mode %d needs S with ldS >= n_sum = %d", int(mode), handle->n_sum);
    const double* cols[ELFI_B200_USERSIM_P_MAX] = {};
    if (simulates) {
        ELFI_REQUIRE(theta_cols_host != nullptr, "usersim_launch: theta_cols_host is NULL");
        for (int j = 0; j < handle->p; ++j) {
            ELFI_REQUIRE(theta_cols_host[j] != nullptr, "usersim_launch: parameter column %d is NULL", j);
            cols[j] = theta_cols_host[j];
        }
    }
    if (B == 0) return ELFI_B200_OK;
    return elfi::run_on_device(ctx, stream, [&](cudaStream_t s) {
        // the kernel's first parameter is UsersimColumns<p>: the first p pointers of cols
        void* args[] = {cols, &B, &key, &offset, &Y, &ldY, &S, &ldS};
        const dim3 grid(unsigned((B + elfi::kUsersimBlock - 1) / elfi::kUsersimBlock));
        ELFI_CUDA_OK(cudaLaunchKernel(reinterpret_cast<const void*>(handle->kernel[mode]), grid,
                                      dim3(elfi::kUsersimBlock), args, 0, s));
        return ELFI_B200_OK;
    });
}

int elfi_b200_usersim_release(elfi_b200_ctx* ctx, elfi_b200_usersim* handle) {
    ELFI_REQUIRE(ctx != nullptr && handle != nullptr, "usersim_release: ctx and handle must not be NULL");
    elfi_b200_usersim** link = &ctx->usersims;
    while (*link && *link != handle) link = &(*link)->next;
    ELFI_REQUIRE(*link != nullptr, "usersim_release: the handle is not one of this context's");
    if (--handle->refs > 0) return ELFI_B200_OK;
    *link = handle->next;
    ELFI_CUDA_OK(cudaSetDevice(ctx->device));
    cudaDeviceSynchronize();   // no launch of the library may still be queued
    elfi::usersim_free(handle);
    return ELFI_B200_OK;
}

}  // extern "C"
