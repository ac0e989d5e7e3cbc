// hd.cuh -- the qualifier of the functions that both the kernels and the g++ harnesses under
// tests/harness compile, so it includes no CUDA header.
#pragma once

#if defined(__CUDACC__)
#define ELFI_HD __host__ __device__ __forceinline__
#define ELFI_UNROLL _Pragma("unroll")
#else
#define ELFI_HD inline
#define ELFI_UNROLL
#endif
