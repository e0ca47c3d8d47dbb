// hd.h — per-thread device logic is written as BM2_HD functions so that the very same source can
// be compiled by g++ into the TEST-ONLY host emulation (tests/host_emul), which checks the kernels'
// control logic against the oracle on a machine without a GPU.  The product never runs this on CPU.
#pragma once
#include <stdint.h>
#if defined(__CUDACC__)
#define BM2_HD __host__ __device__ __forceinline__
#define BM2_D __device__ __forceinline__
#else
#define BM2_HD inline
#define BM2_D inline
#endif

#if defined(__CUDA_ARCH__)
#define BM2_POPC32(x) __popc(x)
#define BM2_POPC64(x) __popcll(x)
#else
#define BM2_POPC32(x) __builtin_popcount(x)
#define BM2_POPC64(x) __builtin_popcountll(x)
#endif

#if defined(__CUDA_ARCH__)
#define BM2_SYNCWARP() __syncwarp()
#define BM2_LDG64(p) ((uint64_t) __ldg(reinterpret_cast<const unsigned long long *>(p)))
#else
#define BM2_SYNCWARP() do {} while (0)
#define BM2_LDG64(p) (*reinterpret_cast<const uint64_t *>(p))
#endif

template <class T> BM2_HD T bm2_min(T a, T b) { return a < b ? a : b; }
template <class T> BM2_HD T bm2_max(T a, T b) { return a > b ? a : b; }
template <class T> BM2_HD void bm2_swap(T &a, T &b) { T t = a; a = b; b = t; }
