// Device helpers shared by the detection decoders (postprocess.cu: the 3-D anchor head and RetinaNet; centernet.cu: MonoFlex and KM3D):
// the sort key, one block sort, torchvision's IoU test and one greedy NMS sweep.
#pragma once
#include <cuda_runtime.h>

#include "common.cuh"

namespace vd3d {

// fp32 ops rounded one at a time: the decoders build without -fmad=false, so the operations that decide index sets say it explicitly
__device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }

// torch CPU sigmoid: 1 / (1 + exp(-x))
__device__ __forceinline__ float sigmoid_ref(float x) { return __fdiv_rn(1.0f, add(1.0f, expf(-x))); }

// The 64-bit sort key of a candidate: ascending key order is (score desc, index asc), torchvision's stable descending sort of the
// index-ordered candidates.  The score must be >= +0, where its bit pattern is monotone.
__device__ __forceinline__ unsigned long long score_key(float score, unsigned int index) {
    return ((unsigned long long)(~__float_as_uint(score)) << 32) | index;
}
__device__ __forceinline__ float key_score(unsigned long long key) { return __uint_as_float(~(unsigned int)(key >> 32)); }
__device__ __forceinline__ unsigned int key_index(unsigned long long key) { return (unsigned int)(key & 0xffffffffu); }

// Ascending bitonic sort of key[0, n) in shared memory, n a power of two, by a block of kThreads threads; with kPayload, pay[i] moves
// with key[i].  Called by the whole block after key[] (and pay[]) are written and synchronised; ends synchronised.
template <int kThreads, bool kPayload>
__device__ __forceinline__ void block_sort(unsigned long long* key, int* pay, int n) {
    const int t = threadIdx.x;
    for (int k = 2; k <= n; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = t; i < n; i += kThreads) {
                int ixj = i ^ j;
                if (ixj > i) {
                    bool up = ((i & k) == 0);
                    unsigned long long a = key[i], c = key[ixj];
                    if ((a > c) == up) {
                        key[i] = c; key[ixj] = a;
                        if (kPayload) { int s0 = pay[i]; pay[i] = pay[ixj]; pay[ixj] = s0; }
                    }
                }
            }
            __syncthreads();
        }
    }
}

// torchvision's CPU nms, in its operation order: areas = (x2 - x1) * (y2 - y1); inter = max(0, xx2 - xx1) * max(0, yy2 - yy1);
// ovr = inter / (area_i + area_j - inter); box j is suppressed by box i if the float ovr > the double threshold.
__device__ __forceinline__ float box_area(float4 b) { return mul(sub(b.z, b.x), sub(b.w, b.y)); }

__device__ __forceinline__ bool iou_above(float4 bi, float ai, float4 bj, float aj, double thr) {
    float xx1 = fmaxf(bi.x, bj.x), yy1 = fmaxf(bi.y, bj.y);
    float xx2 = fminf(bi.z, bj.z), yy2 = fminf(bi.w, bj.w);
    float ww = fmaxf(0.f, sub(xx2, xx1)), hh = fmaxf(0.f, sub(yy2, yy1));
    float inter = mul(ww, hh);
    float ovr = __fdiv_rn(inter, sub(add(ai, aj), inter));
    return (double)ovr > thr;
}

// Greedy class-agnostic NMS over the n <= 4096 sorted boxes box[0, n) with areas area[0, n): box i is kept iff no earlier KEPT box
// suppresses it.  64 rows at a time: all threads build the suppression bit matrix of the block in mask[64][wpr] (bit j of word w of row r:
// box 64w + j comes after row box i and iou_above(i, 64w + j); wpr >= ceil(n / 64) words per row), then warp 0 walks the 64 rows in order
// with the removed set held as one 64-bit word per lane (words l and l + 32).  Writes the sorted positions of the kept boxes, in order,
// to keep[] and returns their count to every thread.  Called by the whole block of kThreads threads after box[] and area[] are
// synchronised; ends synchronised.
template <int kThreads>
__device__ __forceinline__ int nms_sweep(const float4* box, const float* area, int n, int wpr, double thr, unsigned long long* mask,
                                         int* keep) {
    __shared__ int s_nkeep;
    const int t = threadIdx.x;
    const int nw = (n + 63) >> 6;
    unsigned long long removed0 = 0, removed1 = 0;
    int nkeep = 0;
    const int warp = t >> 5, lane = t & 31;
    for (int c = 0; c < nw; ++c) {
        const int words = nw - c;
        for (int e = t; e < 64 * words; e += kThreads) {
            const int r = e & 63, w = c + (e >> 6);
            const int i = c * 64 + r;
            unsigned long long bits = 0;
            if (i < n) {
                const float4 bi = box[i];
                const float ai = area[i];
                const int j0 = w * 64;
                const int jend = min(64, n - j0);
                for (int j = (w == c ? r + 1 : 0); j < jend; ++j)
                    if (iou_above(bi, ai, box[j0 + j], area[j0 + j], thr)) bits |= 1ull << j;
            }
            mask[r * wpr + w] = bits;
        }
        __syncthreads();
        if (warp == 0) {
            const int rows = min(64, n - c * 64);
            for (int r = 0; r < rows; ++r) {
                const unsigned long long rc = c < 32 ? __shfl_sync(0xffffffffu, removed0, c) : __shfl_sync(0xffffffffu, removed1, c - 32);
                if ((rc >> r) & 1ull) continue;                       // warp-uniform
                if (lane == 0) keep[nkeep] = c * 64 + r;
                ++nkeep;
                if (lane >= c && lane < nw) removed0 |= mask[r * wpr + lane];
                if (lane + 32 >= c && lane + 32 < nw) removed1 |= mask[r * wpr + lane + 32];
            }
        }
        __syncthreads();
    }
    if (t == 0) s_nkeep = nkeep;
    __syncthreads();
    return s_nkeep;
}

}  // namespace vd3d
