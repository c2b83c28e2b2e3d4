// Rotated bird's-eye-view box overlap / IoU and NMS (R/lib/ops/iou3d): boxes are [x1, y1, x2, y2, ry].
//
// The overlap area is rotated_overlap.cuh's (shared with km3d_loss.cu).  NMS is fully on the device: a 64 x 64-tile suppression
// bitmask kernel followed by a single-warp greedy sweep (the reference copies the mask to the host and sweeps there,
// iou3d.cpp:87-116).
#include "common.cuh"
#include "rotated_overlap.cuh"

namespace vd3d {

__device__ __forceinline__ float rotated_iou(const float* a, const float* b) {
    float sa = (a[2] - a[0]) * (a[3] - a[1]), sb = (b[2] - b[0]) * (b[3] - b[1]);
    float so = rotated_overlap(a, b);
    return so / fmaxf(sa + sb - so, IOU_EPS);
}

__device__ __forceinline__ float aligned_iou(const float* a, const float* b) {
    float l = fmaxf(a[0], b[0]), r = fminf(a[2], b[2]), t = fmaxf(a[1], b[1]), bt = fminf(a[3], b[3]);
    float w = fmaxf(r - l, 0.f), h = fmaxf(bt - t, 0.f);
    float inter = w * h;
    float sa = (a[2] - a[0]) * (a[3] - a[1]), sb = (b[2] - b[0]) * (b[3] - b[1]);
    return inter / fmaxf(sa + sb - inter, IOU_EPS);
}

template <bool IOU>
__global__ void pairwise_kernel(const float* __restrict__ A, int M, const float* __restrict__ Bx, int N, float* __restrict__ out) {
    int a = blockIdx.y * 16 + threadIdx.y, b = blockIdx.x * 16 + threadIdx.x;
    if (a >= M || b >= N) return;
    float ba[5], bb[5];
#pragma unroll
    for (int i = 0; i < 5; ++i) { ba[i] = A[a * 5 + i]; bb[i] = Bx[b * 5 + i]; }
    out[(long long)a * N + b] = IOU ? rotated_iou(ba, bb) : rotated_overlap(ba, bb);
}

template <bool ROTATED>
__global__ void nms_mask_kernel(const float* __restrict__ boxes, int N, float thr, unsigned long long* __restrict__ mask) {
    const int row = blockIdx.y, col = blockIdx.x;
    const int rows = min(N - row * 64, 64), cols = min(N - col * 64, 64);
    __shared__ float sb[64 * 5];
    if ((int)threadIdx.x < cols)
        for (int i = 0; i < 5; ++i) sb[threadIdx.x * 5 + i] = boxes[(col * 64 + threadIdx.x) * 5 + i];
    __syncthreads();
    if ((int)threadIdx.x < rows) {
        const int cur = row * 64 + threadIdx.x;
        float cb[5];
        for (int i = 0; i < 5; ++i) cb[i] = boxes[cur * 5 + i];
        unsigned long long t = 0;
        int start = (row == col) ? threadIdx.x + 1 : 0;
        for (int i = start; i < cols; ++i) {
            float v = ROTATED ? rotated_iou(cb, sb + i * 5) : aligned_iou(cb, sb + i * 5);
            if (v > thr) t |= 1ULL << i;
        }
        mask[(long long)cur * gridDim.x + col] = t;
    }
}

// greedy sweep over the suppression mask, one warp; keep[] gets the kept indices in order, *count their number
__global__ void nms_sweep_kernel(const unsigned long long* __restrict__ mask, int N, int col_blocks, long long* __restrict__ keep, int* __restrict__ count) {
    extern __shared__ unsigned long long remv[];
    for (int j = threadIdx.x; j < col_blocks; j += 32) remv[j] = 0;
    __syncwarp();
    int n = 0;
    for (int i = 0; i < N; ++i) {
        int nb = i / 64, ib = i % 64;
        if (!(remv[nb] & (1ULL << ib))) {          // uniform across the warp (shared value)
            if (threadIdx.x == 0) keep[n] = i;
            ++n;
            for (int j = nb + threadIdx.x; j < col_blocks; j += 32) remv[j] |= mask[(long long)i * col_blocks + j];
            __syncwarp();
        }
    }
    if (threadIdx.x == 0) *count = n;
}

}  // namespace vd3d

using namespace vd3d;

extern "C" int vd3d_boxes_overlap_bev(const float* a, int M, const float* b, int N, float* out, void* stream) {
    VD3D_REQUIRE(a && b && out && M >= 0 && N >= 0, "boxes_overlap_bev: bad args");
    if (M == 0 || N == 0) return VD3D_OK;
    dim3 grid(cdiv(N, 16), cdiv(M, 16)), block(16, 16);
    pairwise_kernel<false><<<grid, block, 0, (cudaStream_t)stream>>>(a, M, b, N, out);
    VD3D_CHECK_LAUNCH("boxes_overlap_bev");
    return VD3D_OK;
}

extern "C" int vd3d_boxes_iou_bev(const float* a, int M, const float* b, int N, float* out, void* stream) {
    VD3D_REQUIRE(a && b && out && M >= 0 && N >= 0, "boxes_iou_bev: bad args");
    if (M == 0 || N == 0) return VD3D_OK;
    dim3 grid(cdiv(N, 16), cdiv(M, 16)), block(16, 16);
    pairwise_kernel<true><<<grid, block, 0, (cudaStream_t)stream>>>(a, M, b, N, out);
    VD3D_CHECK_LAUNCH("boxes_iou_bev");
    return VD3D_OK;
}

extern "C" long long vd3d_nms_bev_workspace(int N) { return (long long)N * cdiv(N > 0 ? N : 1, 64) * 8 + 64; }

extern "C" int vd3d_nms_bev(const float* boxes, int N, float thresh, int rotated, void* ws, long long* keep, int* count, void* stream) {
    VD3D_REQUIRE(boxes && ws && keep && count && N >= 0, "nms_bev: bad args");
    cudaStream_t st = (cudaStream_t)stream;
    if (N == 0) { VD3D_CUDA(cudaMemsetAsync(count, 0, sizeof(int), st)); return VD3D_OK; }
    int cb = cdiv(N, 64);
    VD3D_REQUIRE(cb * 8 <= 48 * 1024, "nms_bev: too many boxes (%d)", N);
    unsigned long long* mask = (unsigned long long*)ws;
    dim3 grid(cb, cb);
    if (rotated) nms_mask_kernel<true><<<grid, 64, 0, st>>>(boxes, N, thresh, mask);
    else nms_mask_kernel<false><<<grid, 64, 0, st>>>(boxes, N, thresh, mask);
    VD3D_CHECK_LAUNCH("nms_mask");
    nms_sweep_kernel<<<1, 32, cb * sizeof(unsigned long long), st>>>(mask, N, cb, keep, count);
    VD3D_CHECK_LAUNCH("nms_sweep");
    return VD3D_OK;
}
