// usersim_rt.cuh -- the device side of user-written throughput-mode simulators
// (elfi_b200_usersim_compile in usersim.cu, ops.usersim_compile, tools.cuda_simulator).  NVRTC
// compiles this header, then the user's source, then the instantiations of usersim_kernel; the
// user's source sees only what this header declares.
//
// The user defines, at global scope,
//   __device__ void simulate(const double* theta, elfi::RowStream& rng, double* y);
// which writes the n_out doubles y[0 .. n_out) of one row from its p parameters theta[0 .. p) and
// the row's random stream, and, when the simulator has n_sum > 0 summaries,
//   __device__ void summarise(const double* y, double* s);
// which writes the n_sum summaries s[0 .. n_sum) of one row of data.  A missing definition is an
// unresolved function at compile time.
//
// NVRTC's command line defines the salt and the shapes of elfi_b200_usersim_compile:
// ELFI_B200_USERSIM_SALT, and ELFI_B200_USERSIM_P / _N_OUT / _N_SUM, which the source reads as
// elfi::n_params, elfi::n_out and elfi::n_sum.
#pragma once

#if defined(__CUDACC_RTC__)
typedef signed char int8_t;
typedef unsigned char uint8_t;
typedef int int32_t;
typedef unsigned int uint32_t;
typedef long long int64_t;
typedef unsigned long long uint64_t;
#endif

#include "boxmuller.cuh"
#include "philox.cuh"

namespace elfi {

constexpr int n_params = ELFI_B200_USERSIM_P;
constexpr int n_out = ELFI_B200_USERSIM_N_OUT;
constexpr int n_sum = ELFI_B200_USERSIM_N_SUM;

// The Philox4x32-10 stream of one row, in the convention of the built-in simulators (simulate.cu,
// oracle/streams.py): key = the batch key, block m of row r = philox(r & 0xffffffff, r >> 32, m,
// salt).  block / normal2 / uniform2 address blocks directly; next_normal / next_uniform draw
// blocks 0, 1, 2, ... in order (one counter for both) and return the two values of a block one
// after the other: the first next_normal of a row is n0 of block 0, the second n1 of block 0.
struct RowStream {
    Philox ph;
    uint32_t r0, r1;
    uint32_t next_block;          // the block the next sequential draw without a spare takes
    bool has_normal, has_uniform;
    double spare_normal, spare_uniform;

    __device__ RowStream(uint64_t key, uint64_t row)
        : ph(key), r0(uint32_t(row)), r1(uint32_t(row >> 32)), next_block(0u), has_normal(false),
          has_uniform(false), spare_normal(0.0), spare_uniform(0.0) {}

    // the four raw 32-bit words of block m
    __device__ __forceinline__ uint4 block(uint32_t m) const {
        return ph(r0, r1, m, ELFI_B200_USERSIM_SALT);
    }
    // the two standard normals of block m (Box-Muller, boxmuller.cuh)
    __device__ __forceinline__ void normal2(uint32_t m, double& n0, double& n1) const {
        elfi::normal2(block(m), n0, n1);
    }
    // the two 53-bit uniforms on (0, 1] of block m: u01(x, y) and u01(z, w) (philox.cuh)
    __device__ __forceinline__ void uniform2(uint32_t m, double& u0, double& u1) const {
        const uint4 r = block(m);
        u0 = u01(r.x, r.y);
        u1 = u01(r.z, r.w);
    }
    __device__ __forceinline__ double next_normal() {
        if (has_normal) {
            has_normal = false;
            return spare_normal;
        }
        double n0;
        normal2(next_block++, n0, spare_normal);
        has_normal = true;
        return n0;
    }
    __device__ __forceinline__ double next_uniform() {
        if (has_uniform) {
            has_uniform = false;
            return spare_uniform;
        }
        double u0;
        uniform2(next_block++, u0, spare_uniform);
        has_uniform = true;
        return u0;
    }
};

}  // namespace elfi

__device__ void simulate(const double* theta, elfi::RowStream& rng, double* y);
__device__ void summarise(const double* y, double* s);

namespace elfi {

// The modes of usersim_kernel, as elfi_b200_usersim_launch numbers them.
enum UsersimMode {
    USERSIM_DATA = 0,        // simulate into row i of Y
    USERSIM_DATA_SUMM = 1,   // simulate into row i of Y, then summarise it into row i of S
    USERSIM_FUSED = 2,       // simulate into a thread-local row, summarise it into row i of S
    USERSIM_SUMMARISE = 3,   // summarise the given row i of Y into row i of S (no simulation)
};

template <int P>
struct UsersimColumns {
    const double* col[P];   // parameter j of row i is col[j][i]
};

// One thread per row: row i of the call is row offset + i of the batch's stream.
template <int P, int N_OUT, int N_SUM, int MODE>
__global__ void __launch_bounds__(128)
usersim_kernel(UsersimColumns<P> theta_cols, int64_t B, uint64_t key, uint64_t offset,
               double* __restrict__ Y, int64_t ldY, double* __restrict__ S, int64_t ldS) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= B) return;
    if constexpr (MODE == USERSIM_SUMMARISE) {
        summarise(Y + i * ldY, S + i * ldS);
    } else {
        double theta[P];
#pragma unroll
        for (int j = 0; j < P; ++j) theta[j] = theta_cols.col[j][i];
        RowStream rng(key, offset + uint64_t(i));
        if constexpr (MODE == USERSIM_FUSED) {
            double y[N_OUT];
            simulate(theta, rng, y);
            summarise(y, S + i * ldS);
        } else {
            double* y = Y + i * ldY;
            simulate(theta, rng, y);
            if constexpr (MODE == USERSIM_DATA_SUMM) summarise(y, S + i * ldS);
        }
    }
}

}  // namespace elfi
