// Training loss of the 3-D anchor head (AnchorBasedDetection3DHead.loss, R/networks/heads/detection_3d_head.py:101-216, 266-339,
// 402-498, with SigmoidFocalLoss / ModifiedSmoothL1Loss from losses.py and calc_iou from R/networks/utils/utils.py:83-100) for sm_90a.
//
// Forward, four launches whatever B and the number of ground truths (no host synchronisation, graph-capturable):
//   memset   per-ground-truth best keys
//   iou_max  per (anchor tile, image): each valid ground truth's max IoU over the masked anchors and the lowest anchor reaching it,
//            as one 64-bit key (iou_bits << 32 | ~anchor) folded in with an integer atomicMax (order-independent, so deterministic)
//   assign   per (anchor tile, image): IoUs recomputed, _assign (thresholds, low-quality matching in ground-truth order), the prior's
//            z_mean > 0 selection, _encode, the focal / smooth-L1 / alpha-BCE terms; per-block partial sums in double, reduced in a
//            fixed order; the per-anchor assignment
//   combine  one block: partials summed in block order per image, then the reference's batch reduction and the per-image factors
//            the backward scales by
// Backward, one launch: every element's derivative recomputed (autograd's on the reference expression) times grad_output.
//
// Compiled with -fmad=false: calc_iou then rounds every product and sum separately, like torch's fp32 elementwise ops, so the
// IoU -- and with it the assignment -- is bit-identical to the reference's.
#include "common.cuh"
#include "loss_common.cuh"

using vd3d::assign_anchor;
using vd3d::cdiv;
using vd3d::focal;
using vd3d::focal_grad;
using vd3d::fold_gt_keys;
using vd3d::load_gts;
using vd3d::log_sigmoid;
using vd3d::sigmoid;

namespace {

constexpr int kThreads = 256;
constexpr int kGtCols = 12;           // compound_annotation: x1 y1 x2 y2, class, cx cy z, w h l, alpha
constexpr int kReg = 12;              // regression outputs per anchor
constexpr int kTerms = 13;            // 12 smooth-L1 terms + the alpha BCE
constexpr int kMaxClasses = 8;
constexpr int kMaxGt = 512;
// partial record per (image, block): cls sum, 13 regression sums, npos_assigned, npos_selected, nneg, number of valid ground truths
constexpr int kRec = 1 + kTerms + 4;
enum { R_CLS = 0, R_REG = 1, R_NPOS = 1 + kTerms, R_NSEL, R_NNEG, R_NGT };
constexpr int kUnmasked = -2;         // assignment of an anchor outside useful_mask

struct Cfg {
    int B, N, C, M, tiles;
    int match_low_quality, gt_max_assign_all;
    float fg, bg, min_iou, gamma;
    float l1_thr, l1_half_alpha, l1_half_inv;   // float32 of 1/alpha, 0.5*alpha, 0.5/alpha
    float bw[kMaxClasses];                      // balance weight per class
    float rw[kTerms];                           // regression_weight
};

__constant__ float kStds[kReg] = {0.1f, 0.1f, 0.2f, 0.2f, 0.1f, 0.1f, 1.f, 1.f, 1.f, 1.f, 1.f, 1.f};

// ---- pass 1: per-ground-truth max IoU over the masked anchors, and the lowest anchor index reaching it ---------------------------
__global__ void __launch_bounds__(kThreads) iou_max_kernel(const float* __restrict__ anchors, const unsigned char* __restrict__ mask,
                                                           const float* __restrict__ ann, Cfg cfg, unsigned long long* __restrict__ gt_key) {
    extern __shared__ float smem[];
    float* s_gt = smem;
    int* s_idx = reinterpret_cast<int*>(s_gt + cfg.M * kGtCols);
    unsigned long long* s_key = reinterpret_cast<unsigned long long*>(s_idx + ((cfg.M + 1) & ~1));
    __shared__ int s_ng;
    const int b = blockIdx.y;
    const int ng = load_gts<kGtCols>(ann + (size_t)b * cfg.M * kGtCols, cfg.M, kGtCols, s_gt, s_idx, &s_ng);
    if (ng == 0) return;
    const int n = blockIdx.x * kThreads + threadIdx.x;
    const bool m = n < cfg.N && mask[(size_t)b * cfg.N + n];
    float a[4] = {0.f, 0.f, 0.f, 0.f};
    if (m) {
        const float4 v = *reinterpret_cast<const float4*>(anchors + (size_t)n * 4);
        a[0] = v.x; a[1] = v.y; a[2] = v.z; a[3] = v.w;
    }
    fold_gt_keys<kGtCols>(a, m, n, ng, s_gt, s_key, gt_key + (size_t)b * cfg.M);
}

// ---- shared by the assignment pass and the backward -----------------------------------------------------------------------------
// _encode: the 12 regression targets and the alpha class of one (anchor, ground truth) pair; ms = anchor_mean_std_3d[n][label]
__device__ __forceinline__ float encode(const float* a, const float* g, const float* ms, float* t) {
    const float px = (a[0] + a[2]) * 0.5f, py = (a[1] + a[3]) * 0.5f, pw = a[2] - a[0], ph = a[3] - a[1];
    const float gx = (g[0] + g[2]) * 0.5f, gy = (g[1] + g[3]) * 0.5f, gw = g[2] - g[0], gh = g[3] - g[1];
    t[0] = (gx - px) / pw;
    t[1] = (gy - py) / ph;
    t[2] = logf(gw / pw);
    t[3] = logf(gh / ph);
    t[4] = (g[5] - px) / pw;
    t[5] = (g[6] - py) / ph;
    t[6] = (g[7] - ms[0]) / ms[1];
    t[7] = (sinf(g[11] * 2.f) - ms[2]) / ms[3];
    t[8] = (cosf(g[11] * 2.f) - ms[4]) / ms[5];
    t[9] = (g[8] - ms[6]) / ms[7];
    t[10] = (g[9] - ms[8]) / ms[9];
    t[11] = (g[10] - ms[10]) / ms[11];
#pragma unroll
    for (int k = 0; k < kReg; ++k) t[k] = t[k] / kStds[k];
    return cosf(g[11]) > 0.f ? 1.f : 0.f;
}

// Per-block state of the assignment pass and the backward: the image's ground truths and (gt_key given) their best keys, in shared memory.
struct GtShared {
    float* gt;
    float* gmax;
    int* garg;
    int ng;
};

__device__ GtShared load_image(const float* ann, const unsigned long long* gt_key, const Cfg& cfg, int b) {
    extern __shared__ float smem[];
    __shared__ int s_ng;
    GtShared s;
    s.gt = smem;
    s.gmax = s.gt + cfg.M * kGtCols;
    s.garg = reinterpret_cast<int*>(s.gmax + cfg.M);
    int* s_idx = s.garg + cfg.M;
    s.ng = load_gts<kGtCols>(ann + (size_t)b * cfg.M * kGtCols, cfg.M, kGtCols, s.gt, s_idx, &s_ng);
    for (int i = threadIdx.x; gt_key && i < s.ng; i += blockDim.x) {
        const unsigned long long k = gt_key[(size_t)b * cfg.M + i];
        s.gmax[i] = __uint_as_float((unsigned)(k >> 32));
        s.garg[i] = (int)~(unsigned)(k & 0xffffffffull);
    }
    __syncthreads();
    return s;
}

// ---- pass 2: assignment, targets and loss terms; per-block partials -------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) assign_loss_kernel(const float* __restrict__ cls, const float* __restrict__ reg,
                                                               const float* __restrict__ anchors, const unsigned char* __restrict__ mask,
                                                               const float* __restrict__ mean_std, const float* __restrict__ ann,
                                                               const unsigned long long* __restrict__ gt_key, Cfg cfg,
                                                               int* __restrict__ assign, double* __restrict__ partial) {
    __shared__ double s_red[kThreads / 32][kRec];
    const int b = blockIdx.y;
    const GtShared s = load_image(ann, gt_key, cfg, b);
    const int n = blockIdx.x * kThreads + threadIdx.x;
    double acc[kRec];
#pragma unroll
    for (int k = 0; k < kRec; ++k) acc[k] = 0.0;
    if (n < cfg.N) {
        const size_t bn = (size_t)b * cfg.N + n;
        int r = kUnmasked;
        if (mask[bn]) {
            r = -1;
            if (s.ng > 0) {
                const float4 av = *reinterpret_cast<const float4*>(anchors + (size_t)n * 4);
                const float a[4] = {av.x, av.y, av.z, av.w};
                r = assign_anchor<kGtCols>(a, n, s.ng, s.gt, s.gmax, s.garg, cfg);
                const float* g = s.gt + (r > 0 ? r - 1 : 0) * kGtCols;
                const int label = r > 0 ? (int)g[4] : 0;
                const float* ms = mean_std + ((size_t)n * cfg.C + label) * 12;
                const bool sel = r > 0 && ms[0] > 0.f;
                acc[R_NPOS] = r > 0;
                acc[R_NSEL] = sel;
                acc[R_NNEG] = r == 0;
                if (r == 0 || sel) {                                  // positives dropped by the prior keep the ignore label
                    const float* x = cls + bn * (cfg.C + 1);
                    for (int c = 0; c < cfg.C; ++c) {
                        float v = focal(x[c], (r > 0 && c == label) ? 1.f : 0.f, cfg.bw[c], cfg.gamma);
                        acc[R_CLS] += v < 1e-5f ? 0.0 : (double)v;
                    }
                }
                if (sel) {
                    float t[kReg];
                    const float ta = encode(a, g, ms, t);
                    const float* p = reg + bn * kReg;
#pragma unroll
                    for (int k = 0; k < kReg; ++k) {
                        const float d = fabsf(t[k] - p[k]);
                        float l = d <= cfg.l1_thr ? cfg.l1_half_alpha * (d * d) : d - cfg.l1_half_inv;
                        if (d <= 0.01f) l = 0.f;
                        acc[R_REG + k] = (double)(l * cfg.rw[k]);
                    }
                    const float xa = cls[bn * (cfg.C + 1) + cfg.C];
                    const float bce = (1.f - ta) * xa - log_sigmoid(xa);     // BCEWithLogitsLoss
                    acc[R_REG + kReg] = (double)(bce * cfg.rw[kReg]);
                }
            }
        }
        assign[bn] = r;
    }
    double v = vd3d::block_partial<kThreads, kRec>(acc, s_red);
    if (threadIdx.x < kRec) {
        if (threadIdx.x == R_NGT) v = s.ng;
        partial[((size_t)b * cfg.tiles + blockIdx.x) * kRec + threadIdx.x] = v;
    }
}

// ---- combine: per-image sums in block order, then the reference's batch reduction -----------------------------------------------
// cls_loss / reg_loss [1]; counts [B][3] = npos_assigned, npos_selected, nneg; factors [B][2] = d loss / d element
// scale of the cls terms and of the regression terms (zero where the image contributes no gradient).
__global__ void combine_kernel(const double* __restrict__ partial, Cfg cfg, float* __restrict__ cls_loss, float* __restrict__ reg_loss,
                               int* __restrict__ counts, float* __restrict__ factors) {
    extern __shared__ double s_img[];            // [B][kRec]
    for (int b = threadIdx.x; b < cfg.B; b += blockDim.x) {
        double v[kRec];
        for (int k = 0; k < kRec; ++k) v[k] = 0.0;
        for (int t = 0; t < cfg.tiles; ++t)
            for (int k = 0; k < R_NGT; ++k) v[k] += partial[((size_t)b * cfg.tiles + t) * kRec + k];
        v[R_NGT] = partial[(size_t)b * cfg.tiles * kRec + R_NGT];
        for (int k = 0; k < kRec; ++k) s_img[b * kRec + k] = v[k];
        counts[b * 3 + 0] = (int)v[R_NPOS];
        counts[b * 3 + 1] = (int)v[R_NSEL];
        counts[b * 3 + 2] = (int)v[R_NNEG];
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    // cls: mean over images of sum / (positives + negatives), the positives counted after the prior's selection unless it dropped all
    float cls_sum = 0.f, wsum = 0.f;
    for (int b = 0; b < cfg.B; ++b) {
        const double* v = s_img + b * kRec;
        const double npos = v[R_NPOS], nsel = v[R_NSEL];
        const bool has_gt = v[R_NGT] > 0;
        const double den = (nsel > 0 ? nsel : npos) + v[R_NNEG];
        const float c = has_gt ? (float)(v[R_CLS] / den) : 0.f;
        cls_sum += c;
        factors[b * 2] = has_gt ? (float)(1.0 / (cfg.B * den)) : 0.f;
        // a regression row per image, except one whose positives the prior dropped; weight = number of ground truths
        if (!(has_gt && npos > 0 && nsel == 0)) wsum += (float)v[R_NGT];
    }
    const float denom = wsum + 1e-6f;
    float reg[kTerms];
    for (int k = 0; k < kTerms; ++k) reg[k] = 0.f;
    for (int b = 0; b < cfg.B; ++b) {
        const double* v = s_img + b * kRec;
        const bool row = v[R_NSEL] > 0;                      // rows of images with no positive (or no ground truth) are zeros
        const float w = (float)v[R_NGT];
        for (int k = 0; k < kTerms; ++k)
            if (row) reg[k] += w * (float)(v[R_REG + k] / v[R_NSEL]) / denom;
        factors[b * 2 + 1] = row ? (float)((double)w / denom / kTerms / v[R_NSEL]) : 0.f;
    }
    float reg_sum = 0.f;
    for (int k = 0; k < kTerms; ++k) reg_sum += reg[k];
    *cls_loss = cls_sum / cfg.B;
    *reg_loss = reg_sum / kTerms;
}

// ---- backward --------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) backward_kernel(const float* __restrict__ cls, const float* __restrict__ reg,
                                                            const float* __restrict__ anchors, const float* __restrict__ mean_std,
                                                            const float* __restrict__ ann, const int* __restrict__ assign, const float* __restrict__ factors,
                                                            const float* __restrict__ grad_out, Cfg cfg, float* __restrict__ grad_cls,
                                                            float* __restrict__ grad_reg) {
    const int b = blockIdx.y;
    const GtShared s = load_image(ann, nullptr, cfg, b);
    const int n = blockIdx.x * kThreads + threadIdx.x;
    if (n >= cfg.N) return;
    const size_t bn = (size_t)b * cfg.N + n;
    const int C1 = cfg.C + 1;
    float* gc = grad_cls + bn * C1;
    float* gr = grad_reg + bn * kReg;
    const int r = assign[bn];
    const float fc = factors[b * 2] * grad_out[0], fr = factors[b * 2 + 1] * grad_out[1];
    const float* g = s.gt + (r > 0 ? r - 1 : 0) * kGtCols;
    const int label = r > 0 ? (int)g[4] : 0;
    const float* ms = mean_std + ((size_t)n * cfg.C + label) * 12;
    const bool sel = r > 0 && ms[0] > 0.f;
    const float* x = cls + bn * C1;
    for (int c = 0; c < cfg.C; ++c) {
        float d = 0.f;
        if (r == 0 || sel) {
            const float t = (r > 0 && c == label) ? 1.f : 0.f;
            if (!(focal(x[c], t, cfg.bw[c], cfg.gamma) < 1e-5f)) d = focal_grad(x[c], t, cfg.bw[c], cfg.gamma) * fc;
        }
        gc[c] = d;
    }
    if (sel && fr != 0.f) {
        const float a[4] = {anchors[n * 4], anchors[n * 4 + 1], anchors[n * 4 + 2], anchors[n * 4 + 3]};
        float t[kReg];
        const float ta = encode(a, g, ms, t);
        const float* p = reg + bn * kReg;
#pragma unroll
        for (int k = 0; k < kReg; ++k) {
            const float diff = t[k] - p[k], d = fabsf(diff);
            float dl = d <= cfg.l1_thr ? cfg.l1_half_alpha * (2.f * d) : 1.f;
            if (d <= 0.01f) dl = 0.f;
            const float sgn = diff > 0.f ? 1.f : (diff < 0.f ? -1.f : 0.f);
            gr[k] = -sgn * dl * cfg.rw[k] * fr;
        }
        gc[cfg.C] = (sigmoid(x[cfg.C]) - ta) * cfg.rw[kReg] * fr;
    } else {
#pragma unroll
        for (int k = 0; k < kReg; ++k) gr[k] = 0.f;
        gc[cfg.C] = 0.f;
    }
}

size_t gt_smem_bytes(int M) { return (size_t)M * (kGtCols + 3) * sizeof(float) + 16; }
size_t iou_smem_bytes(int M) { return (size_t)M * kGtCols * sizeof(float) + ((M + 1) & ~1) * sizeof(int) + (size_t)M * 8; }

int make_cfg(int B, int N, int C, int M, const float* params, int match_low_quality, int gt_max_assign_all, Cfg& cfg) {
    VD3D_REQUIRE(B > 0 && N > 0 && M >= 0 && M <= kMaxGt, "anchor_loss: bad sizes B=%d N=%d M=%d (M <= %d)", B, N, M, kMaxGt);
    VD3D_REQUIRE(C >= 1 && C <= kMaxClasses, "anchor_loss: %d classes, 1..%d supported", C, kMaxClasses);
    VD3D_REQUIRE(params, "anchor_loss: null parameter array");
    cfg.B = B; cfg.N = N; cfg.C = C; cfg.M = M; cfg.tiles = cdiv(N, kThreads);
    cfg.match_low_quality = match_low_quality != 0;
    cfg.gt_max_assign_all = gt_max_assign_all != 0;
    cfg.fg = params[0]; cfg.bg = params[1]; cfg.min_iou = params[2]; cfg.gamma = params[3];
    cfg.l1_thr = params[4]; cfg.l1_half_alpha = params[5]; cfg.l1_half_inv = params[6];
    for (int c = 0; c < kMaxClasses; ++c) cfg.bw[c] = c < C ? params[7 + c] : 0.f;
    for (int k = 0; k < kTerms; ++k) cfg.rw[k] = params[7 + C + k];
    return VD3D_OK;
}

}  // namespace

extern "C" long long vd3d_anchor_loss_workspace_bytes(int B, int N, int M) {
    return vd3d::assign_workspace_bytes<kThreads, kRec>("anchor_loss", B, N, M, kMaxGt);
}

extern "C" int vd3d_anchor_loss_forward(const float* cls, const float* reg, const float* anchors, const unsigned char* mask,
                                        const float* mean_std, const float* ann, int B, int N, int C, int M, const float* params,
                                        int match_low_quality, int gt_max_assign_all, void* workspace, long long workspace_bytes,
                                        int* assign, int* counts, float* factors, float* cls_loss, float* reg_loss, void* stream) {
    Cfg cfg;
    const int rc = make_cfg(B, N, C, M, params, match_low_quality, gt_max_assign_all, cfg);
    if (rc != VD3D_OK) return rc;
    VD3D_REQUIRE(cls && reg && anchors && mask && mean_std && (M == 0 || ann) && workspace && assign && counts && factors && cls_loss && reg_loss,
                 "anchor_loss_forward: null pointer");
    VD3D_REQUIRE(((uintptr_t)anchors & 15) == 0, "anchor_loss_forward: anchors must be 16-byte aligned");
    const vd3d::AssignLayout L = vd3d::assign_layout<kThreads, kRec>(B, N, M);
    VD3D_REQUIRE((size_t)workspace_bytes >= L.total, "anchor_loss_forward: workspace of %lld bytes, %zu needed", workspace_bytes, L.total);
    char* ws = static_cast<char*>(workspace);
    auto* keys = reinterpret_cast<unsigned long long*>(ws + L.keys);
    auto* partial = reinterpret_cast<double*>(ws + L.partial);
    cudaStream_t st = (cudaStream_t)stream;
    const dim3 grid(cfg.tiles, B);
    if (M > 0) {
        VD3D_CUDA(cudaMemsetAsync(keys, 0, (size_t)B * M * 8, st));
        iou_max_kernel<<<grid, kThreads, iou_smem_bytes(M), st>>>(anchors, mask, ann, cfg, keys);
        VD3D_CHECK_LAUNCH("anchor_loss iou_max");
    }
    assign_loss_kernel<<<grid, kThreads, gt_smem_bytes(M), st>>>(cls, reg, anchors, mask, mean_std, ann, keys, cfg, assign, partial);
    VD3D_CHECK_LAUNCH("anchor_loss assign");
    combine_kernel<<<1, 32, (size_t)B * kRec * sizeof(double), st>>>(partial, cfg, cls_loss, reg_loss, counts, factors);
    VD3D_CHECK_LAUNCH("anchor_loss combine");
    return VD3D_OK;
}

extern "C" int vd3d_anchor_loss_backward(const float* cls, const float* reg, const float* anchors, const float* mean_std,
                                         const float* ann, int B, int N, int C, int M, const float* params, const int* assign,
                                         const float* factors, const float* grad_out, float* grad_cls, float* grad_reg, void* stream) {
    Cfg cfg;
    const int rc = make_cfg(B, N, C, M, params, 1, 1, cfg);
    if (rc != VD3D_OK) return rc;
    VD3D_REQUIRE(cls && reg && anchors && mean_std && (M == 0 || ann) && assign && factors && grad_out && grad_cls && grad_reg,
                 "anchor_loss_backward: null pointer");
    backward_kernel<<<dim3(cfg.tiles, B), kThreads, gt_smem_bytes(M), (cudaStream_t)stream>>>(
        cls, reg, anchors, mean_std, ann, assign, factors, grad_out, cfg, grad_cls, grad_reg);
    VD3D_CHECK_LAUNCH("anchor_loss backward");
    return VD3D_OK;
}
