// Shared host/device helpers for libvd3d_b200 (sm_90a: H100).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include "../../include/vd3d_b200.h"

namespace vd3d {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);
// fp16-range guard of the fp16-split tensor-core engine: a device word (one per device, lazily allocated, zero-initialised) that every
// kernel writing fp16 (hi, lo) activation planes ORs to 1 when a value it splits is beyond the fp16 range (|v| >= 65520 -> hi = inf).
// Read and cleared by vd3d_fp16_range_check; the record kernels fold it into the detection count (-2).  nullptr if the allocation failed.
int* fp16_range_flag();
constexpr float kFp16Overflow = 65520.0f;      // smallest magnitude that rounds to +-inf in fp16 (round to nearest even)

#define VD3D_REQUIRE(cond, ...)                                   \
    do {                                                          \
        if (!(cond)) {                                            \
            ::vd3d::set_error(__VA_ARGS__);                       \
            return VD3D_EINVAL;                                   \
        }                                                         \
    } while (0)

#define VD3D_CHECK_LAUNCH(name)                                                     \
    do {                                                                            \
        cudaError_t e__ = cudaGetLastError();                                       \
        if (e__ != cudaSuccess) {                                                   \
            ::vd3d::set_error("%s: launch failed: %s", name, cudaGetErrorString(e__)); \
            return VD3D_ECUDA;                                                      \
        }                                                                           \
        ::vd3d::count_launch();                                                     \
    } while (0)

#define VD3D_CUDA(call)                                                             \
    do {                                                                            \
        cudaError_t e__ = (call);                                                   \
        if (e__ != cudaSuccess) {                                                   \
            ::vd3d::set_error("%s failed: %s", #call, cudaGetErrorString(e__));     \
            return VD3D_ECUDA;                                                      \
        }                                                                           \
    } while (0)

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }
// the least power of two >= v, and >= lo (a power of two)
__host__ __device__ __forceinline__ int next_pow2(int v, int lo = 1) { int p = lo; while (p < v) p <<= 1; return p; }

constexpr int kNumSMs = 132;  // H100 SXM: persistent grids and tile-cost models

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float amax4(float m, const float4& a) { return fmaxf(fmaxf(m, fmaxf(fabsf(a.x), fabsf(a.y))), fmaxf(fabsf(a.z), fabsf(a.w))); }
__device__ __forceinline__ void note_fp16_range(float amax, int* flag) {
    if (flag && !(amax < kFp16Overflow)) atomicOr(flag, 1);      // also true for NaN
}

}  // namespace vd3d
