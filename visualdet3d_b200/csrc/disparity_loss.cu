// Stereo3D's disparity loss (DisparityLoss(max_disp) -> StereoFocalLoss.loss_per_level -> LaplaceDisp2Prob.getProb,
// R/networks/heads/losses.py:122-135 and R/networks/lib/disparity_loss/*.py) for sm_90a, at the settings the detector ships
// (start_disp 0, dilation 1, one level, focal_coefficient 0, variance 0.5, a label at the cost volume's H, W).
//
// With x = cost [B][D][H][W] (D = max_disp), d = label [B][H][W] and N = B*H*W:
//   outer = 0 < d < D          the loss mask
//   inner = 0 < d < D - 1      Disp2Prob's own mask (end_disp = D - 1)
//   p_c   = softmax_c(-|c - d*inner| / 0.5) * inner + 1e-40      (1e-40 is a float32 subnormal: the build does not flush it)
//   L     = -(1/N) sum_pixels outer * sum_c p_c * log_softmax(x)_c
//   dL/dx_c = -(g * outer / N) * (p_c - softmax(x)_c * sum_c' p_c')
// With no outer pixel in the batch the reference switches to a zero target; every term above is then multiplied by outer = 0, so the
// loss and the gradient are 0 without a batch-wide test.
//
// The Laplace target needs no exp per channel: with k = floor(d), f = d - k, p_c = bl * e^(-2 (k - c)) for c <= k and
// br * e^(-2 (c - k - 1)) above, where bl = e^(-2f - smax) / Z, br = e^(-2(1-f) - smax) / Z and Z (the softmax's denominator) is the sum
// of two geometric series.  e^(-2j) comes from a per-block table in shared memory, so a channel costs one table read and one FMA.
//
// Forward, two launches (no memset, no float atomics, no host synchronisation):
//   pixels   threads over (pixel, image), one thread per pixel walking its D channels at stride H*W, so every warp load is 128
//            contiguous bytes.  An online log-sum-exp (running max m, sum of e^(x - m)) and sum_c p_c (x_c - m), re-based when m moves,
//            so a uniform offset of the logits (+1000) cancels nothing.  Writes each pixel's lse (read by the backward) and one float64
//            partial per block.  Pixels outside outer read no logit.
//   combine  one block: the partials summed in a fixed order, times -1/N.
// Backward, one launch: the same threads read x, the label and lse and write every gradient element once (exact zeros outside outer).
// The incoming gradient is read from device memory, so forward + backward can be captured in a CUDA graph.
//
// A non-finite label makes the loss NaN (the reference raises after a host check); its pixel's gradient is zero.
#include "common.cuh"

using vd3d::cdiv;

namespace {

constexpr int kThreads = 256;
constexpr int kMaxDisp = 1024;         // channels: the shared e^(-2j) table holds D + 1 entries
constexpr int kBatch = 8;              // channel loads a thread issues back to back
constexpr float kEps = 1e-40f;         // Disp2Prob.eps

// A pixel's Laplace target: p_c = (c <= k ? bl * R[k - c] : br * R[c - k - 1]) + eps; bl = br = 0 outside inner (p_c = eps).
struct Target {
    float bl, br;
    int k;
};

__device__ __forceinline__ Target laplace_target(float d, bool inner, int D, const float* R) {
    Target t{0.f, 0.f, 0};
    if (inner) {
        const float kf = floorf(d);
        const float f = d - kf;                           // exact, and so is 1 - f
        const float smax = -2.f * fminf(f, 1.f - f);      // the largest -|c - d| / 0.5, at the channel nearest d
        const float el = expf(-2.f * f - smax), er = expf(-2.f * (1.f - f) - smax);
        t.k = (int)kf;                                    // 0 <= k <= D - 2
        // Z = el * sum_{j <= k} e^(-2j) + er * sum_{j < D - 1 - k} e^(-2j);  sum_{j < n} e^(-2j) = (1 - R[n]) / (1 - e^-2)
        const float z = (el * (1.f - R[t.k + 1]) + er * (1.f - R[D - 1 - t.k])) / (1.f - R[1]);
        t.bl = el / z;
        t.br = er / z;
    }
    return t;
}

__device__ __forceinline__ float target_at(const Target& t, int c, const float* R) {
    const int j = c - t.k;
    return fmaf(j <= 0 ? t.bl : t.br, R[j <= 0 ? -j : j - 1], kEps);
}

__device__ __forceinline__ void fill_table(float* R, int D) {
    for (int j = threadIdx.x; j <= D; j += blockDim.x) R[j] = expf(-2.f * (float)j);
    __syncthreads();
}

__device__ __forceinline__ void label_masks(float d, int D, bool& outer, bool& inner) {
    outer = d > 0.f && d < (float)D;
    inner = d > 0.f && d < (float)(D - 1);
}

// Sum of a double over the block in a fixed order (butterfly within each warp, then warp 0 over the warps in index order).
__device__ __forceinline__ double block_sum(double v, double* red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double s = 0.0;
    if (threadIdx.x == 0)
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w];
    return s;
}

__global__ void __launch_bounds__(kThreads) forward_kernel(const float* __restrict__ x, const float* __restrict__ label, int D, int HW,
                                                           float* __restrict__ lse, double* __restrict__ part) {
    __shared__ float R[kMaxDisp + 1];
    __shared__ double red[kThreads / 32];
    fill_table(R, D);
    const int b = blockIdx.y;
    const int p = blockIdx.x * kThreads + threadIdx.x;
    double acc = 0.0;
    if (p < HW) {
        const size_t pix = (size_t)b * HW + p;
        const float d = __ldg(label + pix);
        bool outer, inner;
        label_masks(d, D, outer, inner);
        acc = (double)(d - d);                            // NaN for a non-finite label: the loss's signal
        float l = 0.f;
        if (outer) {
            const Target t = laplace_target(d, inner, D, R);
            const float* q = x + (size_t)b * D * HW + p;
            float m = __ldg(q);
            float s = 1.f;                                // sum_c e^(x_c - m)
            float P = target_at(t, 0, R);                 // sum_c p_c
            float A = 0.f;                                // sum_c p_c (x_c - m)
            q += HW;
            for (int c0 = 1; c0 < D; c0 += kBatch) {
                float v[kBatch];
#pragma unroll
                for (int i = 0; i < kBatch; ++i) v[i] = c0 + i < D ? __ldg(q + (size_t)i * HW) : 0.f;
                q += (size_t)kBatch * HW;
#pragma unroll
                for (int i = 0; i < kBatch; ++i) {
                    if (c0 + i < D) {
                        const float pc = target_at(t, c0 + i, R);
                        if (v[i] > m) {                   // re-base on the new max
                            s = fmaf(s, expf(m - v[i]), 1.f);
                            A = fmaf(P, m - v[i], A);
                            m = v[i];
                        } else {
                            s += expf(v[i] - m);
                        }
                        A = fmaf(pc, v[i] - m, A);
                        P += pc;
                    }
                }
            }
            const float ls = logf(s);
            l = m + ls;
            acc += (double)fmaf(-P, ls, A);               // sum_c p_c log_softmax(x)_c
        }
        lse[pix] = l;
    }
    const double s = block_sum(acc, red);
    if (threadIdx.x == 0) part[(size_t)blockIdx.y * gridDim.x + blockIdx.x] = s;
}

__global__ void __launch_bounds__(kThreads) combine_kernel(const double* __restrict__ part, int n, double inv_n, float* __restrict__ loss) {
    __shared__ double red[kThreads / 32];
    double a = 0.0;
    for (int i = threadIdx.x; i < n; i += kThreads) a += part[i];
    const double s = block_sum(a, red);
    if (threadIdx.x == 0) *loss = (float)(-s * inv_n);
}

__global__ void __launch_bounds__(kThreads) backward_kernel(const float* __restrict__ x, const float* __restrict__ label,
                                                            const float* __restrict__ lse, int D, int HW, float inv_n,
                                                            const float* __restrict__ grad_loss, float* __restrict__ grad) {
    __shared__ float R[kMaxDisp + 1];
    fill_table(R, D);
    const int b = blockIdx.y;
    const int p = blockIdx.x * kThreads + threadIdx.x;
    if (p >= HW) return;
    const size_t pix = (size_t)b * HW + p;
    const float d = __ldg(label + pix);
    bool outer, inner;
    label_masks(d, D, outer, inner);
    const Target t = laplace_target(d, inner, D, R);
    const float gp = -__ldg(grad_loss) * inv_n;           // d/d (p_c log_softmax_c) at an outer pixel
    const float gP = gp * (inner ? 1.f : (float)D * kEps);  // ... times sum_c p_c
    const float l = outer ? __ldg(lse + pix) : 0.f;
    const float* q = x + (size_t)b * D * HW + p;
    float* o = grad + (size_t)b * D * HW + p;
    for (int c0 = 0; c0 < D; c0 += kBatch) {
        float v[kBatch];
#pragma unroll
        for (int i = 0; i < kBatch; ++i) v[i] = outer && c0 + i < D ? __ldg(q + (size_t)i * HW) : 0.f;
#pragma unroll
        for (int i = 0; i < kBatch; ++i) {
            if (c0 + i < D) {
                const float gc = fmaf(-expf(v[i] - l), gP, gp * target_at(t, c0 + i, R));
                o[(size_t)i * HW] = outer ? gc : 0.f;
            }
        }
        q += (size_t)kBatch * HW;
        o += (size_t)kBatch * HW;
    }
}

int blocks_x(int H, int W) { return cdiv((long long)H * W, kThreads); }

int check_sizes(const char* who, int B, int D, int H, int W) {
    VD3D_REQUIRE(B > 0 && D >= 2 && D <= kMaxDisp && H > 0 && W > 0, "%s: bad sizes B=%d D=%d H=%d W=%d (2 <= D <= %d)", who, B, D, H, W,
                 kMaxDisp);
    VD3D_REQUIRE(B <= 65535, "%s: B = %d images, at most 65535 supported", who, B);
    VD3D_REQUIRE((long long)H * W < (1ll << 31) - kThreads, "%s: H*W = %lld pixels, fewer than 2^31 - %d supported", who, (long long)H * W,
                 kThreads);
    return VD3D_OK;
}

}  // namespace

extern "C" long long vd3d_disparity_loss_workspace_bytes(int B, int D, int H, int W) {
    const int rc = check_sizes("disparity_loss_workspace_bytes", B, D, H, W);
    if (rc != VD3D_OK) return rc;
    return (long long)B * blocks_x(H, W) * (long long)sizeof(double);
}

extern "C" int vd3d_disparity_loss_forward(const float* cost, const float* disp, int B, int D, int H, int W, void* workspace,
                                           long long workspace_bytes, float* lse, float* loss, void* stream) {
    const int rc = check_sizes("disparity_loss_forward", B, D, H, W);
    if (rc != VD3D_OK) return rc;
    VD3D_REQUIRE(cost && disp && workspace && lse && loss, "disparity_loss_forward: null pointer");
    const int bx = blocks_x(H, W);
    const long long need = (long long)B * bx * (long long)sizeof(double);
    VD3D_REQUIRE(workspace_bytes >= need, "disparity_loss_forward: workspace of %lld bytes, %lld needed", workspace_bytes, need);
    auto* part = static_cast<double*>(workspace);
    cudaStream_t st = (cudaStream_t)stream;
    forward_kernel<<<dim3(bx, B), kThreads, 0, st>>>(cost, disp, D, H * W, lse, part);
    VD3D_CHECK_LAUNCH("disparity_loss forward");
    combine_kernel<<<1, kThreads, 0, st>>>(part, B * bx, 1.0 / ((double)B * H * W), loss);
    VD3D_CHECK_LAUNCH("disparity_loss combine");
    return VD3D_OK;
}

extern "C" int vd3d_disparity_loss_backward(const float* cost, const float* disp, const float* lse, int B, int D, int H, int W,
                                            const float* grad_loss, float* grad_cost, void* stream) {
    const int rc = check_sizes("disparity_loss_backward", B, D, H, W);
    if (rc != VD3D_OK) return rc;
    VD3D_REQUIRE(cost && disp && lse && grad_loss && grad_cost, "disparity_loss_backward: null pointer");
    backward_kernel<<<dim3(blocks_x(H, W), B), kThreads, 0, (cudaStream_t)stream>>>(cost, disp, lse, D, H * W,
                                                                                     (float)(1.0 / ((double)B * H * W)), grad_loss,
                                                                                     grad_cost);
    VD3D_CHECK_LAUNCH("disparity_loss backward");
    return VD3D_OK;
}
