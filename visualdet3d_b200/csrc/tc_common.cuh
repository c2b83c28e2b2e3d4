// wgmma / TMA / mbarrier PTX wrappers and the tensor-map encoder shared by the tensor-core kernels (conv2d_tc.cu, psm_tc.cu, ...).
#pragma once
#include "common.cuh"
#include "wgmma.cuh"
#include <cuda.h>
#include <cuda_fp16.h>
#include <mutex>

namespace vd3d {

// ----------------------------------------------------------------------------------------------------------------
// PTX wrappers
// ----------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// Bounded wait: a protocol bug traps (cudaErrorLaunchFailure on the host) after ~2 s instead of hanging the GPU.  (No printf here: a call
// inside the consumers' wait would make the compiler serialise every in-flight wgmma.)
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    uint32_t done = 0, spins = 0;
    long long t0 = 0;
    while (true) {
        asm volatile(
            "{\n\t"
            ".reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t"
            "}\n" : "=r"(done) : "r"(addr), "r"(parity) : "memory");
        if (done) break;
        if ((++spins & 0xFFFu) == 0) {
            const long long t = clock64();
            if (t0 == 0) t0 = t;
            else if (t - t0 > 4000000000LL) __trap();
        }
    }
}
// non-blocking: has the phase of the given parity completed?
__device__ __forceinline__ bool mbar_test(uint64_t* bar, uint32_t parity) {
    uint32_t done;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}\n" : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return done != 0;
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(dst)),
        "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
        "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
// 1-D bulk copy of `bytes` (a multiple of 16, both addresses 16-byte aligned) from global to shared memory, completing on `bar`
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes),
                 "r"(smem_u32(bar)) : "memory");
}
// one elected lane of a fully converged warp (the compiler knows exactly one thread runs the guarded code)
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "elect.sync _|p, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}\n" : "=r"(pred));
    return pred != 0;
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// `count` arrivals at once
__device__ __forceinline__ void mbar_arrive(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
// Programmatic dependent launch (VD3D_PDL=1): a kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may become resident while its
// predecessor is still draining; everything it does before pdl_wait() (barrier init) overlaps the predecessor's tail, and
// pdl_wait() returns when the predecessor has completed and its writes are visible.  Both are no-ops in an ordinary launch.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// shared-memory matrix descriptor of wgmma (sm_90): start address, leading / stride byte offsets (16-byte units), layout type in bits 62..63
// `layout`: the swizzle written by TMA, encoded as the 3-bit field at bit 61: 2 = SWIZZLE_128B (128-byte rows, 8-row groups 1024 B apart),
// 4 = SWIZZLE_64B (64-byte rows, 512 B), 0 = none -- i.e. the 2-bit wgmma layout type (1, 2, 0) shifted to bit 62
__device__ __forceinline__ uint64_t make_sdesc(uint32_t saddr, uint32_t sbo = 1024, uint32_t layout = 2) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFF);        // start address
    d |= (uint64_t)0 << 16;                          // leading byte offset (unused for swizzled K-major)
    d |= (uint64_t)(sbo >> 4) << 32;                 // stride byte offset between 8-row groups (dense: 8 rows * row bytes)
    d |= (uint64_t)layout << 61;
    return d;
}
// K-major, no-swizzle descriptor: 8-row x 16-byte core matrices, `lbo` bytes between core matrices adjacent in K, `sbo` between those adjacent in M / N
__device__ __forceinline__ uint64_t make_sdesc_ns(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo >> 4) & 0x3FFF) << 32;
    return d;
}

// ---- warpgroup MMA (wgmma): four consecutive warps issue together; the accumulator lives in their registers ----
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// pins the accumulator registers at this point of the instruction stream (reads after a wg_wait must not be hoisted above it)
template <int R> __device__ __forceinline__ void wg_fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// Writes the fp32 fragment of a 64 x N accumulator (warpgroup `wg` = rows 64 wg .. 64 wg + 63 of the tile) into a row-major [128][ld] shared-memory
// tile: the per-pixel epilogues read their rows back from there.  `swz` = 7: unpadded rows (ld = N, a multiple of 32) whose 16-byte chunk j of
// row r sits at chunk j ^ (r & 7), which keeps these stores and the epilogue's row reads free of bank conflicts; 0: plain (padded) rows.
template <int N> __device__ __forceinline__ void wg_stage(const float (&d)[N / 2], float* tile, int ld, int wg, int warp, int lane, int swz = 0) {
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
    int sw = r0 & swz;                                   // (rows r0 and r0 + 8 share it)
    if (swz) asm volatile("" : "+r"(sw));                // opaque per call: the N / 4 swizzled offsets are not hoisted out of the caller's tile loop
                                                         // and kept live (spilled) through its MMAs
#pragma unroll
    for (int j = 0; j < N / 8; ++j) {
        const int col = (((2 * j + (c0 >> 2)) ^ sw) << 2) + (c0 & 3);
        *reinterpret_cast<float2*>(tile + r0 * ld + col) = make_float2(d[4 * j], d[4 * j + 1]);
        *reinterpret_cast<float2*>(tile + (r0 + 8) * ld + col) = make_float2(d[4 * j + 2], d[4 * j + 3]);
    }
}
// named barrier of the 256 consumer threads (warps 0..7) of the tensor-core kernels
__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 2, 256;" ::: "memory"); }

// ----------------------------------------------------------------------------------------------------------------
// host: tensor maps (driver entry point fetched at run time: the library does not link libcuda)
// ----------------------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    });
    return fn;
}

// 2-D fp16 map over a [rows][row_pitch] matrix whose first `cols` columns are addressable; box = 64 columns (one 128-byte swizzle row) x box_rows
inline int make_map_2d_h16(CUtensorMap* m, const void* base, long long rows, int cols, long long row_pitch_elems, int box_rows, const char* what) {
    EncodeTiledFn enc = get_encode();
    if (!enc) { set_error("%s: cuTensorMapEncodeTiled unavailable", what); return VD3D_ECUDA; }
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)row_pitch_elems * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
    cuuint32_t es[2] = {1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("%s: cuTensorMapEncodeTiled failed: %d", what, (int)r); return VD3D_ECUDA; }
    return VD3D_OK;
}

}  // namespace vd3d
