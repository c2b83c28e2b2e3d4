// Training loss of the RetinaNet head (RetinanetHead.loss, R/networks/heads/retinanet_head.py:309-362, with _assign / _sample / _encode /
// _decode at 99-255, SigmoidFocalLoss / IoULoss from losses.py:11-46, 93-120 and calc_iou from R/networks/utils/utils.py:83-100) for
// sm_90a.
//
// Forward, four launches whatever B, the number of ground truths or of positives (no host synchronisation, graph-capturable):
//   memset   per-ground-truth best keys
//   iou_max  per (anchor tile, image): each valid ground truth's max IoU over all anchors and the lowest anchor reaching it, folded into
//            one 64-bit key with an integer atomicMax (loss_common.cuh: fold_gt_keys)
//   assign   per (anchor tile, image): IoUs recomputed, _assign, the C focal terms of the one-hot targets, and at positives _encode, the
//            _decode of the prediction and of the encoded target, and the IoU loss; per-block partial sums in double, reduced in a fixed
//            order; the per-anchor assignment
//   combine  one block: partials summed in block order, the batch's positive count, the two 0-d losses and the backward's scale
// Backward, one launch: every element's derivative recomputed from the saved assignment (autograd's on the reference expression) times
// the scale and grad_output.
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

namespace {

constexpr int kThreads = 256;
constexpr int kGtCols = 5;            // the annotation columns the loss reads: x1 y1 x2 y2, class
constexpr int kMaxClasses = 64;
constexpr int kMaxGt = 512;
// partial record per (image, block): focal sum, IoU-loss sum, positives, negatives, positives whose class lies outside [0, C)
constexpr int kRec = 5;
enum { R_CLS = 0, R_REG, R_NPOS, R_NNEG, R_NBAD };
constexpr float kIouEps = 1e-8f;      // IoULoss's eps

struct Cfg {
    int B, N, C, M, K, tiles;
    int match_low_quality, gt_max_assign_all;
    float fg, bg, min_iou, gamma;
    float mean[4], std[4];                      // target_means, target_stds
    float bw[kMaxClasses];                      // balance weight per class
};

// the label of a positive: class.long() when it lies in [0, C), else -1 (the loss is then NaN; the reference's label scatter fails from C up
// and below -C, and wraps -C..-1 into column C + class)
__device__ __forceinline__ int label_of(float cls, int C) { return cls > -1.f && cls < (float)C ? (int)cls : -1; }

// _encode of one (anchor, ground truth) pair
__device__ __forceinline__ void encode(const float* a, const float* g, const Cfg& cfg, float* t) {
    const float px = (a[0] + a[2]) * 0.5f, py = (a[1] + a[3]) * 0.5f, pw = a[2] - a[0], ph = a[3] - a[1];
    const float gx = (g[0] + g[2]) * 0.5f, gy = (g[1] + g[3]) * 0.5f, gw = g[2] - g[0], gh = g[3] - g[1];
    t[0] = (gx - px) / pw;
    t[1] = (gy - py) / ph;
    t[2] = logf(gw / pw);
    t[3] = logf(gh / ph);
#pragma unroll
    for (int k = 0; k < 4; ++k) t[k] = (t[k] - cfg.mean[k]) / cfg.std[k];
}

// _decode of one anchor's deltas d into x1 y1 x2 y2; e[2]: exp of the denormalised dw, dh (the backward's exp derivative)
__device__ __forceinline__ void decode(const float* a, const float* d, const Cfg& cfg, float* box, float* e) {
    float dd[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) dd[k] = d[k] * cfg.std[k] + cfg.mean[k];
    const float px = (a[0] + a[2]) * 0.5f, py = (a[1] + a[3]) * 0.5f, pw = a[2] - a[0], ph = a[3] - a[1];
    e[0] = expf(dd[2]);
    e[1] = expf(dd[3]);
    const float gw = pw * e[0], gh = ph * e[1];
    const float gx = px + pw * dd[0], gy = py + ph * dd[1];
    box[0] = gx - gw * 0.5f;
    box[1] = gy - gh * 0.5f;
    box[2] = gx + gw * 0.5f;
    box[3] = gy + gh * 0.5f;
}

// IoULoss of one (prediction, target) box pair; with g != nullptr, g[0..3] = d loss / d prediction box (autograd's: a max / min tie
// splits 0.5 / 0.5, clamp passes the gradient at its bound, 0 below the eps clamp)
__device__ __forceinline__ float iou_loss(const float* p, const float* t, float* g) {
    const float lt0 = fmaxf(p[0], t[0]), lt1 = fmaxf(p[1], t[1]);
    const float rb0 = fminf(p[2], t[2]), rb1 = fminf(p[3], t[3]);
    const float w0 = rb0 - lt0, w1 = rb1 - lt1;
    const float wc0 = fmaxf(w0, 0.f), wc1 = fmaxf(w1, 0.f);
    const float overlap = wc0 * wc1;
    const float ap = (p[2] - p[0]) * (p[3] - p[1]);
    const float ag = (t[2] - t[0]) * (t[3] - t[1]);
    const float uni = ((ap + ag) - overlap) + kIouEps;
    const float iou = overlap / uni;
    const float iouc = fmaxf(iou, kIouEps);
    if (g) {
        const float g_iou = iou >= kIouEps ? -1.f / iouc : 0.f;
        const float g_un = -g_iou * overlap / (uni * uni);
        const float g_ov = g_iou / uni - g_un;
        const float g_w0 = w0 >= 0.f ? g_ov * wc1 : 0.f, g_w1 = w1 >= 0.f ? g_ov * wc0 : 0.f;
        auto sel = [](float a, float b) { return a > b ? 1.f : (a == b ? 0.5f : 0.f); };      // d max(a, b) / d a
        const float hp = p[3] - p[1], wp = p[2] - p[0];
        g[0] = -g_w0 * sel(p[0], t[0]) - g_un * hp;
        g[1] = -g_w1 * sel(p[1], t[1]) - g_un * wp;
        g[2] = g_w0 * sel(t[2], p[2]) + g_un * hp;
        g[3] = g_w1 * sel(t[3], p[3]) + g_un * wp;
    }
    return -logf(iouc);
}

// Per-block state of the assignment pass and the backward: the image's ground truths and (gt_key given) their best keys, in shared memory.
struct GtShared {
    float* gt;
    float* gmax;
    int* garg;
    int ng;
};

__device__ GtShared load_image(const float* ann, const unsigned long long* gt_key, const Cfg& cfg, int b) {
    extern __shared__ __align__(16) float smem[];
    __shared__ int s_ng;
    GtShared s;
    s.gt = smem;
    s.gmax = s.gt + cfg.M * kGtCols;
    s.garg = reinterpret_cast<int*>(s.gmax + cfg.M);
    int* s_idx = s.garg + cfg.M;
    s.ng = load_gts<kGtCols>(ann + (size_t)b * cfg.M * cfg.K, cfg.M, cfg.K, s.gt, s_idx, &s_ng);
    for (int i = threadIdx.x; gt_key && i < s.ng; i += blockDim.x) {
        const unsigned long long k = gt_key[(size_t)b * cfg.M + i];
        s.gmax[i] = __uint_as_float((unsigned)(k >> 32));
        s.garg[i] = (int)~(unsigned)(k & 0xffffffffull);
    }
    __syncthreads();
    return s;
}

__device__ __forceinline__ void load_anchor(const float* anchors, int n, float* a) {
    const float4 v = *reinterpret_cast<const float4*>(anchors + (size_t)n * 4);
    a[0] = v.x; a[1] = v.y; a[2] = v.z; a[3] = v.w;
}

// ---- pass 1: per-ground-truth max IoU over all anchors, and the lowest anchor index reaching it ------------------------------------
__global__ void __launch_bounds__(kThreads) iou_max_kernel(const float* __restrict__ anchors, const float* __restrict__ ann, Cfg cfg,
                                                           unsigned long long* __restrict__ gt_key) {
    // the 64-bit keys first: s_gt holds 5 floats per row, so after it an odd M would leave them 4 bytes off the 8-byte boundary their
    // 64-bit stores and atomics need
    extern __shared__ __align__(16) float smem[];
    unsigned long long* s_key = reinterpret_cast<unsigned long long*>(smem);
    float* s_gt = smem + 2 * cfg.M;
    int* s_idx = reinterpret_cast<int*>(s_gt + cfg.M * kGtCols);
    __shared__ int s_ng;
    const int b = blockIdx.y;
    const int ng = load_gts<kGtCols>(ann + (size_t)b * cfg.M * cfg.K, cfg.M, cfg.K, s_gt, s_idx, &s_ng);
    if (ng == 0) return;
    const int n = blockIdx.x * kThreads + threadIdx.x;
    const bool m = n < cfg.N;
    float a[4] = {0.f, 0.f, 0.f, 0.f};
    if (m) load_anchor(anchors, n, a);
    fold_gt_keys<kGtCols>(a, m, n, ng, s_gt, s_key, gt_key + (size_t)b * cfg.M);
}

// ---- pass 2: assignment, focal and IoU terms; per-block partials ----------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) assign_loss_kernel(const float* __restrict__ cls, const float* __restrict__ reg,
                                                               const float* __restrict__ anchors, const float* __restrict__ ann,
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
        float a[4];
        load_anchor(anchors, n, a);
        // an image without a valid row: _assign makes every anchor negative
        const int r = s.ng > 0 ? assign_anchor<kGtCols>(a, n, s.ng, s.gt, s.gmax, s.garg, cfg) : 0;
        acc[R_NPOS] = r > 0;
        acc[R_NNEG] = r == 0;
        if (r >= 0) {                                                 // ignored anchors (-1 in every column) contribute zero
            const float* g = s.gt + (r > 0 ? r - 1 : 0) * kGtCols;
            const int label = r > 0 ? label_of(g[4], cfg.C) : -1;
            if (r > 0 && label < 0) acc[R_NBAD] = 1.0;
            const float* x = cls + bn * cfg.C;
            for (int c = 0; c < cfg.C; ++c) {
                const float v = focal(x[c], c == label ? 1.f : 0.f, cfg.bw[c], cfg.gamma);
                acc[R_CLS] += v < 1e-5f ? 0.0 : (double)v;
            }
            if (r > 0) {
                float t[4], pb[4], tb[4], e[2];
                encode(a, g, cfg, t);
                decode(a, reg + bn * 4, cfg, pb, e);
                decode(a, t, cfg, tb, e);                             // the target's round trip, as the reference decodes it
                acc[R_REG] = (double)iou_loss(pb, tb, nullptr);
            }
        }
        assign[bn] = r;
    }
    double v = vd3d::block_partial<kThreads, kRec>(acc, s_red);
    if (threadIdx.x < kRec) {
        partial[((size_t)b * cfg.tiles + blockIdx.x) * kRec + threadIdx.x] = v;
    }
}

// ---- combine: per-image sums in block order, then the batch reduction -------------------------------------------------------------
// cls_loss / reg_loss 0-d; counts [B][3] = positives, negatives, ignored; scale [1] = d loss / d element of both sums, 1 / (P + 1e-4)
// with P the batch's positive count; NaN losses and scale when a positive's class lies outside [0, C).
__global__ void combine_kernel(const double* __restrict__ partial, Cfg cfg, float* __restrict__ cls_loss, float* __restrict__ reg_loss,
                               int* __restrict__ counts, float* __restrict__ scale) {
    extern __shared__ double s_img[];            // [B][kRec]
    for (int b = threadIdx.x; b < cfg.B; b += blockDim.x) {
        double v[kRec];
        for (int k = 0; k < kRec; ++k) v[k] = 0.0;
        for (int t = 0; t < cfg.tiles; ++t)
            for (int k = 0; k < kRec; ++k) v[k] += partial[((size_t)b * cfg.tiles + t) * kRec + k];
        for (int k = 0; k < kRec; ++k) s_img[b * kRec + k] = v[k];
        counts[b * 3 + 0] = (int)v[R_NPOS];
        counts[b * 3 + 1] = (int)v[R_NNEG];
        counts[b * 3 + 2] = cfg.N - (int)v[R_NPOS] - (int)v[R_NNEG];
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    double cls = 0.0, reg = 0.0, npos = 1e-4, bad = 0.0;      // number_of_positives starts at 1e-4 (retinanet_head.py:315)
    for (int b = 0; b < cfg.B; ++b) {
        const double* v = s_img + b * kRec;
        cls += v[R_CLS];
        reg += v[R_REG];
        npos += v[R_NPOS];
        bad += v[R_NBAD];
    }
    const float nan = __int_as_float(0x7fffffff);
    *cls_loss = bad > 0 ? nan : (float)(cls / npos);
    *reg_loss = bad > 0 ? nan : (float)(reg / npos);
    *scale = bad > 0 ? nan : (float)(1.0 / npos);
}

// ---- backward --------------------------------------------------------------------------------------------------------------------
// Every element is its derivative times the scale and grad_out, zeros included, so a NaN scale makes every gradient NaN.
__global__ void __launch_bounds__(kThreads) backward_kernel(const float* __restrict__ cls, const float* __restrict__ reg,
                                                            const float* __restrict__ anchors, const float* __restrict__ ann,
                                                            const int* __restrict__ assign, const float* __restrict__ scale,
                                                            const float* __restrict__ grad_out, Cfg cfg, float* __restrict__ grad_cls,
                                                            float* __restrict__ grad_reg) {
    const int b = blockIdx.y;
    const GtShared s = load_image(ann, nullptr, cfg, b);
    const int n = blockIdx.x * kThreads + threadIdx.x;
    if (n >= cfg.N) return;
    const size_t bn = (size_t)b * cfg.N + n;
    const int r = assign[bn];
    const float fc = scale[0] * grad_out[0], fr = scale[0] * grad_out[1];
    const float* g = s.gt + (r > 0 ? r - 1 : 0) * kGtCols;
    const int label = r > 0 ? label_of(g[4], cfg.C) : -1;
    const float* x = cls + bn * cfg.C;
    float* gc = grad_cls + bn * cfg.C;
    for (int c = 0; c < cfg.C; ++c) {
        float d = 0.f;
        if (r >= 0) {
            const float t = c == label ? 1.f : 0.f;
            if (!(focal(x[c], t, cfg.bw[c], cfg.gamma) < 1e-5f)) d = focal_grad(x[c], t, cfg.bw[c], cfg.gamma);
        }
        gc[c] = d * fc;
    }
    float gp[4] = {0.f, 0.f, 0.f, 0.f};
    if (r > 0) {
        float a[4], t[4], pb[4], tb[4], e[2], et[2], gb[4];
        load_anchor(anchors, n, a);
        encode(a, g, cfg, t);
        decode(a, reg + bn * 4, cfg, pb, e);
        decode(a, t, cfg, tb, et);
        iou_loss(pb, tb, gb);
        // back through _decode: x1 / x2 = gx -/+ gw * 0.5, gx = px + pw * dx, gw = pw * exp(dw), d = pred * std + mean
        const float pw = a[2] - a[0], ph = a[3] - a[1];
        const float g_gx = gb[0] + gb[2], g_gy = gb[1] + gb[3];
        const float g_gw = (gb[2] - gb[0]) * 0.5f, g_gh = (gb[3] - gb[1]) * 0.5f;
        gp[0] = g_gx * pw * cfg.std[0];
        gp[1] = g_gy * ph * cfg.std[1];
        gp[2] = g_gw * pw * e[0] * cfg.std[2];
        gp[3] = g_gh * ph * e[1] * cfg.std[3];
    }
    *reinterpret_cast<float4*>(grad_reg + bn * 4) = make_float4(gp[0] * fr, gp[1] * fr, gp[2] * fr, gp[3] * fr);
}

size_t gt_smem_bytes(int M) { return (size_t)M * (kGtCols + 3) * sizeof(float) + 16; }
size_t iou_smem_bytes(int M) { return (size_t)M * 8 + (size_t)M * kGtCols * sizeof(float) + (size_t)M * sizeof(int); }

// params: fg, bg, min_iou, gamma, target_means[4], target_stds[4], the balance weight of each class
int make_cfg(int B, int N, int C, int M, int K, const float* params, int match_low_quality, int gt_max_assign_all, Cfg& cfg) {
    VD3D_REQUIRE(B > 0 && N > 0 && M >= 0 && M <= kMaxGt && K >= kGtCols, "retina_loss: bad sizes B=%d N=%d M=%d K=%d (M <= %d, K >= %d)",
                 B, N, M, K, kMaxGt, kGtCols);
    VD3D_REQUIRE(C >= 1 && C <= kMaxClasses, "retina_loss: %d classes, 1..%d supported", C, kMaxClasses);
    VD3D_REQUIRE(params, "retina_loss: null parameter array");
    cfg.B = B; cfg.N = N; cfg.C = C; cfg.M = M; cfg.K = K; cfg.tiles = cdiv(N, kThreads);
    cfg.match_low_quality = match_low_quality != 0;
    cfg.gt_max_assign_all = gt_max_assign_all != 0;
    cfg.fg = params[0]; cfg.bg = params[1]; cfg.min_iou = params[2]; cfg.gamma = params[3];
    for (int k = 0; k < 4; ++k) {
        cfg.mean[k] = params[4 + k];
        cfg.std[k] = params[8 + k];
    }
    for (int c = 0; c < kMaxClasses; ++c) cfg.bw[c] = c < C ? params[12 + c] : 0.f;
    return VD3D_OK;
}

}  // namespace

extern "C" long long vd3d_retina_loss_workspace_bytes(int B, int N, int M) {
    return vd3d::assign_workspace_bytes<kThreads, kRec>("retina_loss", B, N, M, kMaxGt);
}

extern "C" int vd3d_retina_loss_forward(const float* cls, const float* reg, const float* anchors, const float* ann, int B, int N, int C,
                                        int M, int K, const float* params, int match_low_quality, int gt_max_assign_all, void* workspace,
                                        long long workspace_bytes, int* assign, int* counts, float* scale, float* cls_loss, float* reg_loss,
                                        void* stream) {
    Cfg cfg;
    const int rc = make_cfg(B, N, C, M, K, params, match_low_quality, gt_max_assign_all, cfg);
    if (rc != VD3D_OK) return rc;
    VD3D_REQUIRE(cls && reg && anchors && (M == 0 || ann) && workspace && assign && counts && scale && cls_loss && reg_loss,
                 "retina_loss_forward: null pointer");
    VD3D_REQUIRE(((uintptr_t)anchors & 15) == 0, "retina_loss_forward: anchors must be 16-byte aligned");
    const vd3d::AssignLayout L = vd3d::assign_layout<kThreads, kRec>(B, N, M);
    VD3D_REQUIRE((size_t)workspace_bytes >= L.total, "retina_loss_forward: workspace of %lld bytes, %zu needed", workspace_bytes, L.total);
    char* ws = static_cast<char*>(workspace);
    auto* keys = reinterpret_cast<unsigned long long*>(ws + L.keys);
    auto* partial = reinterpret_cast<double*>(ws + L.partial);
    cudaStream_t st = (cudaStream_t)stream;
    const dim3 grid(cfg.tiles, B);
    if (M > 0) {
        VD3D_CUDA(cudaMemsetAsync(keys, 0, (size_t)B * M * 8, st));
        iou_max_kernel<<<grid, kThreads, iou_smem_bytes(M), st>>>(anchors, ann, cfg, keys);
        VD3D_CHECK_LAUNCH("retina_loss iou_max");
    }
    assign_loss_kernel<<<grid, kThreads, gt_smem_bytes(M), st>>>(cls, reg, anchors, ann, keys, cfg, assign, partial);
    VD3D_CHECK_LAUNCH("retina_loss assign");
    combine_kernel<<<1, 32, (size_t)B * kRec * sizeof(double), st>>>(partial, cfg, cls_loss, reg_loss, counts, scale);
    VD3D_CHECK_LAUNCH("retina_loss combine");
    return VD3D_OK;
}

extern "C" int vd3d_retina_loss_backward(const float* cls, const float* reg, const float* anchors, const float* ann, int B, int N, int C,
                                         int M, int K, const float* params, const int* assign, const float* scale, const float* grad_out,
                                         float* grad_cls, float* grad_reg, void* stream) {
    Cfg cfg;
    const int rc = make_cfg(B, N, C, M, K, params, 1, 1, cfg);
    if (rc != VD3D_OK) return rc;
    VD3D_REQUIRE(cls && reg && anchors && (M == 0 || ann) && assign && scale && grad_out && grad_cls && grad_reg,
                 "retina_loss_backward: null pointer");
    VD3D_REQUIRE(((uintptr_t)anchors & 15) == 0 && ((uintptr_t)grad_reg & 15) == 0,
                 "retina_loss_backward: anchors and grad_reg must be 16-byte aligned");
    backward_kernel<<<dim3(cfg.tiles, B), kThreads, gt_smem_bytes(M), (cudaStream_t)stream>>>(
        cls, reg, anchors, ann, assign, scale, grad_out, cfg, grad_cls, grad_reg);
    VD3D_CHECK_LAUNCH("retina_loss backward");
    return VD3D_OK;
}
