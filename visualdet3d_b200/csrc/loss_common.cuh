// Device helpers shared by the training-loss kernels (anchor_loss.cu, retina_loss.cu, monoflex_loss.cu, km3d_loss.cu).
#pragma once
#include <cuda_runtime.h>

#include "common.cuh"

namespace vd3d {

// ---- fixed-order reductions: no float atomics, so two runs give the same bits -------------------------------------------------------

// One block's sums of the kRec per-thread accumulators (float or double, summed in double): a shuffle tree per warp, then the warps in
// index order.  s_red: [kThreads / 32][kRec] of shared scratch.  Called by the whole block; thread k < kRec gets slot k's sum (the others 0).
template <int kThreads, int kRec, class T>
__device__ __forceinline__ double block_partial(const T (&acc)[kRec], double (*s_red)[kRec]) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < kRec; ++k) {
        double v = acc[k];
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
        if (lane == 0) s_red[warp][k] = v;
    }
    __syncthreads();
    double v = 0.0;
    if (threadIdx.x < kRec)
        for (int w = 0; w < kThreads / 32; ++w) v += s_red[w][threadIdx.x];
    return v;
}

// The sum of p[i * stride], i < n, over one warp: lane-strided, then a shuffle tree; every lane gets it.
__device__ inline double warp_sum(const double* p, int n, int stride, int lane) {
    double v = 0.0;
    for (int i = lane; i < n; i += 32) v += p[(size_t)i * stride];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    return __shfl_sync(0xffffffffu, v, 0);
}

// torch.nn.functional.logsigmoid, in its overflow-free form
__device__ __forceinline__ float log_sigmoid(float x) { return fminf(x, 0.f) - log1pf(expf(-fabsf(x))); }
__device__ __forceinline__ float sigmoid(float x) { return 1.f / (1.f + expf(-x)); }
// torch.sign: 0 at 0
__device__ __forceinline__ float sign0(float x) { return x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f); }

// ---- anchor assignment of the anchor heads (_assign, detection_3d_head.py:101-171 and retinanet_head.py:99-171, textually identical) --
// Both callers compile with -fmad=false, so calc_iou rounds like torch's fp32 elementwise ops and the assignment is the reference's.

// calc_iou(a, b) (R/networks/utils/utils.py:83-100), one pair, the reference's expression order
__host__ __device__ __forceinline__ float calc_iou(const float* a, const float* b) {
    const float area = (b[2] - b[0]) * (b[3] - b[1]);
    float iw = fminf(a[2], b[2]) - fmaxf(a[0], b[0]);
    float ih = fminf(a[3], b[3]) - fmaxf(a[1], b[1]);
    iw = fmaxf(iw, 0.f);
    ih = fmaxf(ih, 0.f);
    float ua = ((a[2] - a[0]) * (a[3] - a[1]) + area) - iw * ih;
    ua = fmaxf(ua, 1e-8f);
    const float inter = iw * ih;
    return inter / ua;
}

// calc_iou of float32 anchors against float64 boxes, as torch promotes it: the anchor's coordinates widen exactly, its own area is still
// rounded in float32, everything else is float64.  Callers compile with -fmad=false.
__host__ __device__ __forceinline__ double calc_iou(const float* a, const double* b) {
    const double area = (b[2] - b[0]) * (b[3] - b[1]);
    double iw = fmin((double)a[2], b[2]) - fmax((double)a[0], b[0]);
    double ih = fmin((double)a[3], b[3]) - fmax((double)a[1], b[1]);
    iw = fmax(iw, 0.0);
    ih = fmax(ih, 0.0);
    double ua = ((double)((a[2] - a[0]) * (a[3] - a[1])) + area) - iw * ih;
    ua = fmax(ua, 1e-8);
    const double inter = iw * ih;
    return inter / ua;
}

// The image's valid ground-truth rows (column 4, the class, != -1) of ann_b [M][pitch], compacted in their original order into
// s_gt[ng][kCols] (each row's first kCols columns).  s_idx: M ints of shared scratch.  Called by the whole block; returns ng.
template <int kCols>
__device__ int load_gts(const float* ann_b, int M, int pitch, float* s_gt, int* s_idx, int* s_ng) {
    if (threadIdx.x < 32) {
        int base = 0;
        for (int m0 = 0; m0 < M; m0 += 32) {
            const int m = m0 + (int)threadIdx.x;
            const bool valid = m < M && ann_b[(size_t)m * pitch + 4] != -1.f;
            const unsigned bal = __ballot_sync(0xffffffffu, valid);
            if (valid) s_idx[base + __popc(bal & ((1u << threadIdx.x) - 1u))] = m;
            base += __popc(bal);
        }
        if (threadIdx.x == 0) *s_ng = base;
    }
    __syncthreads();
    const int ng = *s_ng;
    for (int k = threadIdx.x; k < ng * kCols; k += blockDim.x) s_gt[k] = ann_b[(size_t)s_idx[k / kCols] * pitch + k % kCols];
    __syncthreads();
    return ng;
}

// Each of the ng ground truths' max IoU over this block's taking-part anchors, and the lowest anchor index reaching it, folded into
// gt_key[i] as one 64-bit key (iou_bits << 32 | ~anchor) with an integer atomicMax: order-independent, so deterministic.  a: the thread's
// anchor n, m: whether it takes part.  s_key: ng slots of shared scratch.  Called by the whole block (ng > 0).
template <int kCols>
__device__ __forceinline__ void fold_gt_keys(const float* a, bool m, int n, int ng, const float* s_gt, unsigned long long* s_key,
                                             unsigned long long* gt_key) {
    for (int i = threadIdx.x; i < ng; i += blockDim.x) s_key[i] = 0ull;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    for (int i = 0; i < ng; ++i) {
        const unsigned bits = m ? __float_as_uint(calc_iou(a, s_gt + i * kCols)) : 0u;       // IoU >= 0: bit order is value order
        const unsigned mx = __reduce_max_sync(0xffffffffu, bits);
        const unsigned idx = __reduce_min_sync(0xffffffffu, (m && bits == mx) ? (unsigned)n : 0xffffffffu);
        if (lane == 0 && idx != 0xffffffffu) atomicMax(s_key + i, ((unsigned long long)mx << 32) | (unsigned long long)(~idx));
    }
    __syncthreads();
    for (int i = threadIdx.x; i < ng; i += blockDim.x)
        if (s_key[i]) atomicMax(gt_key + i, s_key[i]);
}

// _assign for one taking-part anchor: the 1-based compacted ground-truth index, 0 negative, -1 ignored.  s_gmax / s_garg: each ground
// truth's max IoU and first arg anchor (from fold_gt_keys).  Cfg: fg, bg, min_iou, match_low_quality, gt_max_assign_all.
template <int kCols, class Cfg>
__device__ __forceinline__ int assign_anchor(const float* a, int n, int ng, const float* s_gt, const float* s_gmax, const int* s_garg,
                                             const Cfg& cfg) {
    float best = calc_iou(a, s_gt);
    int arg = 0;
    for (int i = 1; i < ng; ++i) {
        const float v = calc_iou(a, s_gt + i * kCols);
        if (v > best) { best = v; arg = i; }                          // first maximum, like max(dim=1)
    }
    int r = -1;
    if (best >= 0.f && best < cfg.bg) r = 0;
    if (best >= cfg.fg) r = arg + 1;
    if (cfg.match_low_quality) {
        for (int i = 0; i < ng; ++i) {                                // ground-truth order: the last match wins
            if (!(s_gmax[i] >= cfg.min_iou)) continue;
            if (cfg.gt_max_assign_all ? calc_iou(a, s_gt + i * kCols) == s_gmax[i] : n == s_garg[i]) r = i + 1;
        }
    }
    return r;
}

// Workspace of the assigning losses: each image's M best keys (fold_gt_keys; zeroed before the IoU pass), then the assignment pass's
// [B][tiles][kRec] double partials at the next 256-byte boundary, tiles = ceil(N / kThreads).
struct AssignLayout {
    size_t keys, partial, total;
};

template <int kThreads, int kRec>
AssignLayout assign_layout(int B, int N, int M) {
    AssignLayout L;
    const size_t tiles = (size_t)cdiv(N, kThreads);
    L.keys = 0;
    L.partial = ((size_t)B * M * 8 + 255) & ~(size_t)255;
    L.total = L.partial + (size_t)B * tiles * kRec * sizeof(double);
    return L;
}

// vd3d_<who>_workspace_bytes: the layout's size, or VD3D_EINVAL for sizes the kernels do not take (at most max_gt rows per image)
template <int kThreads, int kRec>
long long assign_workspace_bytes(const char* who, int B, int N, int M, int max_gt) {
    if (B <= 0 || N <= 0 || M < 0 || M > max_gt) {
        set_error("%s_workspace_bytes: bad sizes B=%d N=%d M=%d", who, B, N, M);
        return VD3D_EINVAL;
    }
    return (long long)assign_layout<kThreads, kRec>(B, N, M).total;
}

// ---- SigmoidFocalLoss (losses.py:11-46) ----------------------------------------------------------------------------------------------
__device__ __forceinline__ float powg(float x, float g) { return g == 2.f ? x * x : powf(x, g); }

// one element for target t in {0, 1} (t = -1 is zero and handled by the caller), before the < 1e-5 clamp
__device__ __forceinline__ float focal(float x, float t, float bw, float gamma) {
    const float p = sigmoid(x);
    const float fw = powg(t == 1.f ? 1.f - p : p, gamma);
    const float bce = -(t * log_sigmoid(x)) * bw - ((1.f - t) * log_sigmoid(-x));
    return fw * bce;
}

// its derivative in x, focal weight not detached (autograd on the reference expression)
__device__ __forceinline__ float focal_grad(float x, float t, float bw, float gamma) {
    const float p = sigmoid(x), q = 1.f - p;
    if (t == 1.f) {
        const float bce = -log_sigmoid(x) * bw;
        const float dfw = gamma == 0.f ? 0.f : gamma * powg(q, gamma - 1.f) * (-p * q);
        return dfw * bce + powg(q, gamma) * (-bw * q);
    }
    const float bce = -log_sigmoid(-x);
    const float dfw = gamma == 0.f ? 0.f : gamma * powg(p, gamma - 1.f) * (p * q);
    return dfw * bce + powg(p, gamma) * p;
}

// ---- the heatmap focal terms of CenterNet-style heads (KM3DHead._neg_loss, km3d_head.py:61-98) -----------------------------------------
constexpr int kHmRec = 3;              // per-block partial: positive sum, negative sum, positive count

__device__ __forceinline__ void hm_terms(float x, float g, float& pos, float& neg) {
    const float p = sigmoid(x);
    pos = neg = 0.f;
    if (g == 1.f && !(p > 0.99f)) pos = log_sigmoid(x) * ((1.f - p) * (1.f - p));
    if (g < 1.f && !(p < 0.01f)) {
        const float w = (1.f - g) * (1.f - g);
        neg = log_sigmoid(-x) * (p * p) * (w * w);
    }
}

// d (pos + neg) / dx, the powers of p not detached
__device__ __forceinline__ float hm_grad(float x, float g) {
    const float p = sigmoid(x), q = 1.f - p;
    if (g == 1.f) return p > 0.99f ? 0.f : q * q * q - 2.f * p * q * q * log_sigmoid(x);
    if (g < 1.f && !(p < 0.01f)) {
        const float w = (1.f - g) * (1.f - g);
        return (w * w) * (-p * p * p + 2.f * p * p * q * log_sigmoid(-x));
    }
    return 0.f;
}

// One block's partials of the focal terms over hm / gt [n]: the block is number `block` of `nblocks` striding over the elements by
// kThreads; the partial (kHmRec doubles) goes to partial[block].  Reduced in a fixed order (warp shuffle tree, then warps in order).
template <int kThreads>
__device__ __forceinline__ void hm_block_partial(const float* __restrict__ hm, const float* __restrict__ gt, long long n, int block,
                                                 int nblocks, double* __restrict__ partial) {
    __shared__ double s_red[kThreads / 32][kHmRec];
    double acc[kHmRec] = {0.0, 0.0, 0.0};
    for (long long i = (long long)block * kThreads + threadIdx.x; i < n; i += (long long)nblocks * kThreads) {
        const float g = gt[i];
        float pos, neg;
        hm_terms(hm[i], g, pos, neg);
        acc[0] += pos;
        acc[1] += neg;
        acc[2] += g == 1.f ? 1.0 : 0.0;
    }
    const double v = block_partial<kThreads, kHmRec>(acc, s_red);
    if (threadIdx.x < kHmRec) partial[(size_t)block * kHmRec + threadIdx.x] = v;
}

// ---- one object row of KM3DHead._RegWeightedL1Loss (km3d_head.py:100-115) -------------------------------------------------------------
// at(c): the keypoint map's channel c at the row's pixel; mask / target: the row's kKp entries of hps_mask / hps; dep: the row's depth,
// transformed on a copy (0.01 dep below 5, log10(dep - 4) + 0.1 from 5).  Returns the row's weighted L1 in l and its mask sum in ms; with
// kGrad, adds d l / d at(c) times scale to g[c].
template <int kKp, bool kGrad, class At>
__device__ __forceinline__ void weighted_l1_row(At at, const unsigned char* mask, const float* target, float dep, float scale, float* g,
                                                float& l_out, float& ms_out) {
    const float dep_t = dep < 5.f ? dep * 0.01f : log10f(dep - 4.f) + 0.1f;
    float l = 0.f, ms = 0.f;
    for (int c = 0; c < kKp; ++c) {
        const float m = (float)mask[c];
        const float d = at(c) * m - target[c] * m;
        if (kGrad) g[c] += sign0(d) * m * dep_t * scale;
        l += fabsf(d);
        ms += m;
    }
    l_out = l * dep_t;
    ms_out = ms;
}

// ---- one object row of compute_rot_loss (rtm3d_utils.py:9-49) -------------------------------------------------------------------------
// at(c): the rotation map's channel c (8) at the row's pixel; valid: the row's reg_mask; bin / res: its rotbin / rotres (2 each).  The two
// cross-entropies use the logits times reg_mask (every row counts); the sin / cos smooth-L1 of bin j counts where bin j is set.  Returns
// the cross-entropy sum in ce and, for each set bin j, its residual loss in res[j] and 1 in n[j] (untouched otherwise); with kGrad, adds
// the gradient (cross-entropy scaled by s_ce, residual j by s_res[j]) to g[0..7].
template <bool kGrad, class At>
__device__ __forceinline__ void rot_row(At at, bool valid, const long long* bin2, const float* res2, float s_ce, float s_res1, float s_res2,
                                        float* g, float& ce_out, float* res, float* n) {
    const float m = valid ? 1.f : 0.f;
    float ce = 0.f;
    for (int j = 0; j < 2; ++j) {
        const long long bin = bin2[j];
        const float z0 = at(4 * j) * m, z1 = at(4 * j + 1) * m;
        const float mx = fmaxf(z0, z1);
        const float lse = mx + logf(expf(z0 - mx) + expf(z1 - mx));
        ce += lse - (bin != 0 ? z1 : z0);
        if (kGrad) {
            g[4 * j] += (expf(z0 - lse) - (bin != 0 ? 0.f : 1.f)) * m * s_ce;
            g[4 * j + 1] += (expf(z1 - lse) - (bin != 0 ? 1.f : 0.f)) * m * s_ce;
        }
        if (bin != 0) {
            const float r = res2[j];
            const float ds = at(4 * j + 2) - sinf(r), dc = at(4 * j + 3) - cosf(r);
            if (kGrad) {
                const float f = j == 0 ? s_res1 : s_res2;
                g[4 * j + 2] += (fabsf(ds) < 1.f ? ds : sign0(ds)) * f;
                g[4 * j + 3] += (fabsf(dc) < 1.f ? dc : sign0(dc)) * f;
            } else {
                const float ads = fabsf(ds), adc = fabsf(dc);
                res[j] = (ads < 1.f ? 0.5f * ds * ds : ads - 0.5f) + (adc < 1.f ? 0.5f * dc * dc : adc - 0.5f);
                n[j] = 1.f;
            }
        }
    }
    ce_out = ce;
}

}  // namespace vd3d
