// Training loss of the MonoFlex head (MonoFlexHead.loss, R/networks/heads/monoflex_head.py:181-236, with KM3DHead._neg_loss /
// _RegWeightedL1Loss / _RotLoss from km3d_head.py:61-130, compute_rot_loss and decode_depth_from_keypoints from
// R/networks/utils/rtm3d_utils.py:9-49, 141-182, and IoULoss from losses.py:93-120) for sm_90a.
//
// Forward, three launches whatever B, K and the number of objects (no memset, no host synchronisation, graph-capturable):
//   hm       grid-stride over B*C*H*W: the heatmap focal terms; per-block partials (positive sum, negative sum, positive count)
//   rows     one block per image, one thread per object row: the maps read at ind in NCHW (no permuted copy), the weighted-L1, rotation
//            and gathered terms; the image's partials reduced in a fixed order
//   combine  one warp: partials summed in a fixed order in float64, the num_pos == 0 choice, the nine terms, the weighted total and the
//            per-term factors the backward scales by
// Backward, one launch: each block owns a tile of one image's pixels and writes every gradient map there in full -- the heatmap
// derivative, and zeros plus, at a gathered pixel, the contributions of the image's rows whose ind is that pixel, summed in row order.
//
// No float atomics anywhere, so two runs give the same bits.  A row whose ind lies outside [0, H*W) is never read; it makes every loss
// (and every factor, so every gradient) NaN.
#include <algorithm>

#include "common.cuh"
#include "loss_common.cuh"

using vd3d::cdiv;
using vd3d::hm_grad;
using vd3d::kHmRec;
using vd3d::log_sigmoid;
using vd3d::sigmoid;
using vd3d::warp_sum;

namespace {

constexpr int kThreads = 256;
constexpr int kMaxRows = 128;          // object rows per image (K)
constexpr int kRowThreads = kMaxRows;
constexpr int kHmBlocksMax = 4 * vd3d::kNumSMs;
constexpr int kTerms = 9;              // hm, hp, box2d, off, dim, depth, kpd, rot, soft_depth: the reference's weight_dict order
__constant__ float kWeight[kTerms] = {1.f, 1.f, 1.f, 0.5f, 1.f, 1.f, 0.2f, 1.f, 0.2f};

// the nine head maps, in the order of the C ABI, and their channel counts
enum { M_HM, M_BBOX2D, M_HPS, M_ROT, M_DIM, M_REG, M_DEPTH, M_DUNC, M_CUNC, kMaps };
__constant__ int kMapCh[kMaps] = {0, 4, 20, 8, 3, 2, 1, 1, 3};
// a row's gradient: the eight gathered maps' channels back to back
constexpr int kGathCh = 42;
__constant__ int kGOff[kMaps] = {0, 0, 4, 24, 32, 35, 37, 38, 39};

// targets, in the order of the C ABI
enum { T_HM, T_IND, T_REG_MASK, T_HPS, T_HPS_MASK, T_DEP, T_ROTBIN, T_ROTRES, T_BOX, T_DIM, T_REG, T_KPMASK, T_P2, kTargets };

// per-image partial record of the rows pass
enum { R_HP, R_HPM, R_CE, R_RES1, R_N1, R_RES2, R_N2, R_N, R_BOX, R_DIM, R_OFF, R_DEPTH, R_KPD, R_SOFT, R_BAD, kRec };
// factors [kFac] f32 written by combine: d term / d (summed element) of each denominator
enum { F_HM, F_HP, F_CE, F_RES1, F_RES2, F_GATH, kFac };

struct Args {
    const float* map[kMaps];
    const float* hm_t;
    const long long* ind;
    const unsigned char* reg_mask;
    const float* hps_t;
    const unsigned char* hps_mask;
    const float* dep;
    const long long* rotbin;
    const float* rotres;
    const float* box_t;
    const float* dim_t;
    const float* reg_t;
    const float* kp_mask;
    const float* P2;
    int B, C, H, W, K, hm_blocks;
    float unc_lo, unc_hi, unc_w;
};

// scales of the backward: d loss / d (summed element) of each term, grad_output included
struct Scales {
    float hm, hp, ce, res1, res2, box, dim, off, depth, kpd, soft;
};

__device__ __forceinline__ float sgn(float x) { return x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f); }
// d max(a, b) / d a and d min(a, b) / d a: a tie splits the gradient
__device__ __forceinline__ float dmax(float a, float b) { return a > b ? 1.f : (a == b ? 0.5f : 0.f); }
__device__ __forceinline__ float dmin(float a, float b) { return a < b ? 1.f : (a == b ? 0.5f : 0.f); }
__device__ __forceinline__ float clampf(float x, float lo, float hi) { return fminf(fmaxf(x, lo), hi); }
__device__ __forceinline__ float clamp_pass(float x, float lo, float hi) { return (x >= lo && x <= hi) ? 1.f : 0.f; }

__global__ void __launch_bounds__(kThreads) hm_kernel(const float* __restrict__ hm, const float* __restrict__ gt, long long n,
                                                      double* __restrict__ partial) {
    vd3d::hm_block_partial<kThreads>(hm, gt, n, blockIdx.x, gridDim.x, partial);
}

// ---- one object row: its loss terms (rec, forward) or its gradient at the gathered pixel (g[kGathCh], backward) ----------------------
// Returns false (and touches nothing but rec[R_BAD]) for an ind outside [0, H*W).
template <bool kGrad>
__device__ bool row_eval(const Args& a, int b, int k, const Scales* s, float* rec, float* g) {
    const int HW = a.H * a.W;
    const size_t r = (size_t)b * a.K + k;
    const long long id = a.ind[r];
    if (id < 0 || id >= HW) {
        if (!kGrad) rec[R_BAD] = 1.f;
        return false;
    }
    auto at = [&](int m, int c) { return a.map[m][((size_t)b * kMapCh[m] + c) * HW + id]; };
    if (kGrad)
        for (int c = 0; c < kGathCh; ++c) g[c] = 0.f;

    // hp_loss: every row, under hps_mask; dep transformed on a copy
    const float dep = a.dep[r];
    {
        float l, ms;
        vd3d::weighted_l1_row<20, kGrad>([&](int c) { return at(M_HPS, c); }, a.hps_mask + r * 20, a.hps_t + r * 20, dep,
                                         kGrad ? s->hp : 0.f, g + kGOff[M_HPS], l, ms);
        if (!kGrad) { rec[R_HP] = l; rec[R_HPM] = ms; }
    }

    // rot_loss: two cross-entropies of every row (logits times reg_mask), smooth-L1 of the rows whose bin is set
    const bool valid = a.reg_mask[r] != 0;
    {
        float ce, res[2] = {0.f, 0.f}, n[2] = {0.f, 0.f};
        vd3d::rot_row<kGrad>([&](int c) { return at(M_ROT, c); }, valid, a.rotbin + r * 2, a.rotres + r * 2, kGrad ? s->ce : 0.f,
                             kGrad ? s->res1 : 0.f, kGrad ? s->res2 : 0.f, g + kGOff[M_ROT], ce, res, n);
        if (!kGrad) {
            rec[R_CE] = ce;
            rec[R_RES1] = res[0]; rec[R_N1] = n[0];
            rec[R_RES2] = res[1]; rec[R_N2] = n[1];
        }
    }
    if (!valid) return true;

    // ---- the gathered terms: rows with reg_mask set ----
    if (!kGrad) rec[R_N] = 1.f;
    // box2d_loss: IoU loss of (-l, -t, r, b) boxes
    {
        float p[4], q[4];
        for (int c = 0; c < 4; ++c) {
            p[c] = c < 2 ? -at(M_BBOX2D, c) : at(M_BBOX2D, c);
            q[c] = c < 2 ? -a.box_t[r * 4 + c] : a.box_t[r * 4 + c];
        }
        const float ltx = fmaxf(p[0], q[0]), lty = fmaxf(p[1], q[1]), rbx = fminf(p[2], q[2]), rby = fminf(p[3], q[3]);
        const float wx = rbx - ltx, wy = rby - lty;
        const float w = fmaxf(wx, 0.f), h = fmaxf(wy, 0.f);
        const float ov = w * h;
        const float ap = (p[2] - p[0]) * (p[3] - p[1]), ag = (q[2] - q[0]) * (q[3] - q[1]);
        const float un = ap + ag - ov + 1e-8f;
        const float iou = ov / un;
        const float ic = fmaxf(iou, 1e-8f);
        if (!kGrad) {
            rec[R_BOX] = -logf(ic);
        } else {
            const float gi = iou >= 1e-8f ? -s->box / ic : 0.f;
            const float gov = gi / un + gi * ov / (un * un);
            const float gap = -gi * ov / (un * un);
            const float gw = wx >= 0.f ? gov * h : 0.f, gh = wy >= 0.f ? gov * w : 0.f;
            float dp[4];
            dp[0] = -gw * dmax(p[0], q[0]) - gap * (p[3] - p[1]);
            dp[1] = -gh * dmax(p[1], q[1]) - gap * (p[2] - p[0]);
            dp[2] = gw * dmin(p[2], q[2]) + gap * (p[3] - p[1]);
            dp[3] = gh * dmin(p[3], q[3]) + gap * (p[2] - p[0]);
            for (int c = 0; c < 4; ++c) g[kGOff[M_BBOX2D] + c] += c < 2 ? -dp[c] : dp[c];
        }
    }
    // dim_loss and off_loss: L1
    {
        float l = 0.f;
        for (int c = 0; c < 3; ++c) {
            const float d = at(M_DIM, c) - a.dim_t[r * 3 + c];
            l += fabsf(d);
            if (kGrad) g[kGOff[M_DIM] + c] += sgn(d) * s->dim;
        }
        if (!kGrad) rec[R_DIM] = l;
        l = 0.f;
        for (int c = 0; c < 2; ++c) {
            const float d = at(M_REG, c) - a.reg_t[r * 2 + c];
            l += fabsf(d);
            if (kGrad) g[kGOff[M_REG] + c] += sgn(d) * s->off;
        }
        if (!kGrad) rec[R_OFF] = l;
    }
    // the depths: direct (exp(-depth)) and from the keypoints (decode_depth_from_keypoints), with their clamped uncertainties
    const float draw = at(M_DEPTH, 0), dd = expf(-draw);
    const float uraw[4] = {at(M_DUNC, 0), at(M_CUNC, 0), at(M_CUNC, 1), at(M_CUNC, 2)};
    float u[4];
    for (int i = 0; i < 4; ++i) u[i] = clampf(uraw[i], a.unc_lo, a.unc_hi);
    const float fh = a.P2[(size_t)b * 12] * at(M_DIM, 1);
    // keypoint heights: centre (kp 8 - kp 9), corner groups 0 ((7, 3) - (0, 4)) and 1 ((2, 6) - (1, 5)); y of keypoint i is channel 2i+1
    constexpr int kTop[5] = {17, 15, 7, 5, 13}, kBot[5] = {19, 1, 9, 3, 11};
    float ht[5], den[5];
    for (int i = 0; i < 5; ++i) {
        ht[i] = at(M_HPS, kTop[i]) - at(M_HPS, kBot[i]);
        den[i] = fmaxf(ht[i], 0.f) * 4.f + 1e-8f;
    }
    const float kraw[3] = {fh / den[0], (fh / den[1] + fh / den[2]) / 2.f, (fh / den[3] + fh / den[4]) / 2.f};
    float kd[3];
    for (int j = 0; j < 3; ++j) kd[j] = clampf(kraw[j], 0.1f, 100.f);
    // soft depth: merged with weights 1 / exp(u), normalised
    const float depths[4] = {dd, kd[0], kd[1], kd[2]};
    float wt[4], wsum = 0.f;
    for (int i = 0; i < 4; ++i) {
        wt[i] = 1.f / expf(u[i]);
        wsum += wt[i];
    }
    float merged = 0.f;
    for (int i = 0; i < 4; ++i) {
        wt[i] = wt[i] / wsum;
        merged += depths[i] * wt[i];
    }
    const float e0 = expf(-u[0]);
    if (!kGrad) {
        rec[R_DEPTH] = fabsf(dd - dep) * e0 + u[0] * a.unc_w;
        float kl = 0.f;
        for (int j = 0; j < 3; ++j) {
            const float l = fabsf(kd[j] - dep) * expf(-u[j + 1]) + u[j + 1] * a.unc_w;
            const float v = a.kp_mask[r * 3 + j];
            kl += l * v + (1.f - v) * l;
        }
        rec[R_KPD] = kl / 3.f;
        rec[R_SOFT] = fabsf(merged - dep);
        return true;
    }
    float gdep[4] = {0.f, 0.f, 0.f, 0.f}, gu[4] = {0.f, 0.f, 0.f, 0.f};
    gdep[0] = sgn(dd - dep) * e0 * s->depth;
    gu[0] = (-fabsf(dd - dep) * e0 + a.unc_w) * s->depth;
    for (int j = 0; j < 3; ++j) {                          // the detached half of the kpd loss carries no gradient
        const float f = a.kp_mask[r * 3 + j] / 3.f * s->kpd, e = expf(-u[j + 1]);
        gdep[j + 1] = sgn(kd[j] - dep) * e * f;
        gu[j + 1] = (-fabsf(kd[j] - dep) * e + a.unc_w) * f;
    }
    const float gm = sgn(merged - dep) * s->soft;
    for (int i = 0; i < 4; ++i) {
        gdep[i] += gm * wt[i];
        gu[i] += gm * (-(depths[i] - merged) * wt[i]);
    }
    g[kGOff[M_DEPTH]] += gdep[0] * -dd;
    g[kGOff[M_DUNC]] += gu[0] * clamp_pass(uraw[0], a.unc_lo, a.unc_hi);
    for (int j = 0; j < 3; ++j) g[kGOff[M_CUNC] + j] += gu[j + 1] * clamp_pass(uraw[j + 1], a.unc_lo, a.unc_hi);
    // through the clamp, the group mean and relu(height) into the keypoint channels; dim[..., 1] is detached
    for (int i = 0; i < 5; ++i) {
        const int j = i == 0 ? 0 : (i + 1) / 2;
        const float gk = gdep[j + 1] * clamp_pass(kraw[j], 0.1f, 100.f) * (i == 0 ? 1.f : 0.5f);
        if (gk != 0.f && ht[i] > 0.f) {
            const float gh = -gk * fh / (den[i] * den[i]) * 4.f;
            g[kGOff[M_HPS] + kTop[i]] += gh;
            g[kGOff[M_HPS] + kBot[i]] -= gh;
        }
    }
    return true;
}

// Args from the C ABI's pointer arrays
Args make_args(const void* const* maps, const void* const* targets, int B, int C, int H, int W, int K, float lo, float hi, float uw) {
    Args a;
    for (int m = 0; m < kMaps; ++m) a.map[m] = static_cast<const float*>(maps[m]);
    a.hm_t = static_cast<const float*>(targets[T_HM]);
    a.ind = static_cast<const long long*>(targets[T_IND]);
    a.reg_mask = static_cast<const unsigned char*>(targets[T_REG_MASK]);
    a.hps_t = static_cast<const float*>(targets[T_HPS]);
    a.hps_mask = static_cast<const unsigned char*>(targets[T_HPS_MASK]);
    a.dep = static_cast<const float*>(targets[T_DEP]);
    a.rotbin = static_cast<const long long*>(targets[T_ROTBIN]);
    a.rotres = static_cast<const float*>(targets[T_ROTRES]);
    a.box_t = static_cast<const float*>(targets[T_BOX]);
    a.dim_t = static_cast<const float*>(targets[T_DIM]);
    a.reg_t = static_cast<const float*>(targets[T_REG]);
    a.kp_mask = static_cast<const float*>(targets[T_KPMASK]);
    a.P2 = static_cast<const float*>(targets[T_P2]);
    a.B = B; a.C = C; a.H = H; a.W = W; a.K = K;
    const long long n = (long long)B * C * H * W;
    a.hm_blocks = (int)std::min<long long>(cdiv(n, kThreads * 8), kHmBlocksMax);
    a.unc_lo = lo; a.unc_hi = hi; a.unc_w = uw;
    return a;
}

// ---- the rows pass: one block per image ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kRowThreads) rows_kernel(Args a, double* __restrict__ partial) {
    __shared__ double s_red[kRowThreads / 32][kRec];
    const int b = blockIdx.x, k = threadIdx.x;
    float rec[kRec];
#pragma unroll
    for (int i = 0; i < kRec; ++i) rec[i] = 0.f;
    if (k < a.K) row_eval<false>(a, b, k, nullptr, rec, nullptr);
    const double v = vd3d::block_partial<kRowThreads, kRec>(rec, s_red);
    if (threadIdx.x < kRec) partial[(size_t)b * kRec + threadIdx.x] = v;
}

// ---- combine: one warp; sums in a fixed order (vd3d::warp_sum: lane-strided, then a shuffle tree) -----------------------------

__global__ void combine_kernel(const double* __restrict__ hm_part, const double* __restrict__ row_part, Args a, float* __restrict__ terms,
                               float* __restrict__ total, float* __restrict__ factors) {
    const int lane = threadIdx.x;
    double hmv[kHmRec], rv[kRec];
    for (int i = 0; i < kHmRec; ++i) hmv[i] = warp_sum(hm_part + i, a.hm_blocks, kHmRec, lane);
    for (int i = 0; i < kRec; ++i) rv[i] = warp_sum(row_part + i, a.B, kRec, lane);
    if (lane != 0) return;
    const float pos = (float)hmv[0], neg = (float)hmv[1], npos = (float)hmv[2];
    float t[kTerms], f[kFac];
    t[0] = npos == 0.f ? -neg : -(pos + neg) / npos;
    f[F_HM] = npos == 0.f ? -1.f : -1.f / npos;
    const float hp_den = (float)rv[R_HPM] + 1e-4f;
    t[1] = (float)rv[R_HP] / hp_den;
    f[F_HP] = 1.f / hp_den;
    const float gath_den = (float)((double)rv[R_N] + 1e-4);
    f[F_GATH] = 1.f / gath_den;
    t[2] = (float)rv[R_BOX] / gath_den;
    t[3] = (float)rv[R_OFF] / gath_den;
    t[4] = (float)rv[R_DIM] / gath_den;
    t[5] = (float)rv[R_DEPTH] / gath_den;
    t[6] = (float)rv[R_KPD] / gath_den;
    const float rows = (float)((long long)a.B * a.K);
    float rot = (float)rv[R_CE] / rows;
    f[F_CE] = 1.f / rows;
    f[F_RES1] = rv[R_N1] > 0 ? 1.f / (float)rv[R_N1] : 0.f;
    f[F_RES2] = rv[R_N2] > 0 ? 1.f / (float)rv[R_N2] : 0.f;
    if (rv[R_N1] > 0) rot += (float)rv[R_RES1] / (float)rv[R_N1];
    if (rv[R_N2] > 0) rot += (float)rv[R_RES2] / (float)rv[R_N2];
    t[7] = rot;
    t[8] = (float)rv[R_SOFT] / gath_den;
    const bool bad = rv[R_BAD] > 0;
    float sum = 0.f;
    for (int i = 0; i < kTerms; ++i) {
        if (bad) t[i] = __int_as_float(0x7fc00000);
        terms[i] = t[i];
        sum = sum + t[i] * kWeight[i];
    }
    *total = sum;
    for (int i = 0; i < kFac; ++i) factors[i] = bad ? __int_as_float(0x7fc00000) : f[i];
}

// ---- backward ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) backward_kernel(Args a, const float* __restrict__ factors, const float* __restrict__ g_terms,
                                                            const float* __restrict__ g_total,
                                                            float* g_hm, float* g_box, float* g_hps, float* g_rot, float* g_dim, float* g_reg,
                                                            float* g_depth, float* g_dunc, float* g_cunc) {
    __shared__ int s_row[kMaxRows];
    __shared__ int s_pix[kMaxRows];
    __shared__ int s_cnt[kMaxRows / 32];
    __shared__ float s_g[kMaxRows][kGathCh];
    const int b = blockIdx.y, HW = a.H * a.W;
    const int p0 = blockIdx.x * kThreads;
    // the image's rows whose ind falls in this tile, compacted in row order
    const int k = threadIdx.x;
    bool hit = false;
    long long id = -1;
    if (k < a.K) {
        id = a.ind[(size_t)b * a.K + k];
        hit = id >= p0 && id < p0 + kThreads && id < HW;
    }
    const unsigned bal = __ballot_sync(0xffffffffu, hit);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (warp < kMaxRows / 32 && lane == 0) s_cnt[warp] = __popc(bal);
    __syncthreads();
    int nm = 0, off = 0;
    for (int w = 0; w < kMaxRows / 32; ++w) {
        if (w < warp) off += s_cnt[w];
        nm += s_cnt[w];
    }
    if (hit) {
        const int slot = off + __popc(bal & ((1u << lane) - 1u));
        s_row[slot] = k;
        s_pix[slot] = (int)id;
    }
    Scales s;
    {
        float gt[kTerms];
        const float gtot = g_total ? *g_total : 0.f;
        for (int i = 0; i < kTerms; ++i) gt[i] = (g_terms ? g_terms[i] : 0.f) + kWeight[i] * gtot;
        s.hm = factors[F_HM] * gt[0];
        s.hp = factors[F_HP] * gt[1];
        s.box = factors[F_GATH] * gt[2];
        s.off = factors[F_GATH] * gt[3];
        s.dim = factors[F_GATH] * gt[4];
        s.depth = factors[F_GATH] * gt[5];
        s.kpd = factors[F_GATH] * gt[6];
        s.ce = factors[F_CE] * gt[7];
        s.res1 = factors[F_RES1] * gt[7];
        s.res2 = factors[F_RES2] * gt[7];
        s.soft = factors[F_GATH] * gt[8];
    }
    __syncthreads();
    if (threadIdx.x < nm) row_eval<true>(a, b, s_row[threadIdx.x], &s, nullptr, s_g[threadIdx.x]);
    __syncthreads();
    const int p = p0 + threadIdx.x;
    if (p >= HW) return;
    float* const outs[kMaps] = {g_hm, g_box, g_hps, g_rot, g_dim, g_reg, g_depth, g_dunc, g_cunc};
    for (int m = 1; m < kMaps; ++m) {
        for (int c = 0; c < kMapCh[m]; ++c) {
            float v = 0.f;
            for (int i = 0; i < nm; ++i)
                if (s_pix[i] == p) v += s_g[i][kGOff[m] + c];
            outs[m][((size_t)b * kMapCh[m] + c) * HW + p] = v;
        }
    }
    for (int c = 0; c < a.C; ++c) {
        const size_t i = ((size_t)b * a.C + c) * HW + p;
        g_hm[i] = hm_grad(a.map[M_HM][i], a.hm_t[i]) * s.hm;
    }
}

struct Layout {
    size_t hm_part, row_part, factors, total;
};

Layout layout(const Args& a) {
    Layout L;
    L.hm_part = 0;
    L.row_part = ((size_t)a.hm_blocks * kHmRec * sizeof(double) + 255) & ~(size_t)255;
    L.factors = L.row_part + (((size_t)a.B * kRec * sizeof(double) + 255) & ~(size_t)255);
    L.total = L.factors + kFac * sizeof(float);
    return L;
}

int check_sizes(const char* who, int B, int C, int H, int W, int K) {
    VD3D_REQUIRE(B > 0 && C > 0 && H > 0 && W > 0 && K > 0 && K <= kMaxRows, "%s: bad sizes B=%d C=%d H=%d W=%d K=%d (1 <= K <= %d)", who, B,
                 C, H, W, K, kMaxRows);
    VD3D_REQUIRE((long long)H * W < (1ll << 31), "%s: H*W = %lld pixels, at most 2^31 - 1 supported", who, (long long)H * W);
    return VD3D_OK;
}

}  // namespace

extern "C" long long vd3d_monoflex_loss_workspace_bytes(int B, int C, int H, int W, int K) {
    const int rc = check_sizes("monoflex_loss_workspace_bytes", B, C, H, W, K);
    if (rc != VD3D_OK) return rc;
    const void* none[kTargets] = {};
    return (long long)layout(make_args(none, none, B, C, H, W, K, 0.f, 0.f, 0.f)).total;
}

extern "C" int vd3d_monoflex_loss_forward(const void* const* maps, const void* const* targets, int B, int C, int H, int W, int K,
                                          float unc_lo, float unc_hi, float unc_w, void* workspace, long long workspace_bytes, float* terms,
                                          float* total, void* stream) {
    const int rc = check_sizes("monoflex_loss_forward", B, C, H, W, K);
    if (rc != VD3D_OK) return rc;
    VD3D_REQUIRE(maps && targets && workspace && terms && total, "monoflex_loss_forward: null pointer");
    for (int i = 0; i < kMaps; ++i) VD3D_REQUIRE(maps[i], "monoflex_loss_forward: null map %d", i);
    for (int i = 0; i < kTargets; ++i) VD3D_REQUIRE(targets[i], "monoflex_loss_forward: null target %d", i);
    VD3D_REQUIRE(unc_hi >= unc_lo, "monoflex_loss_forward: uncertainty range [%g, %g] is empty", unc_lo, unc_hi);
    const Args a = make_args(maps, targets, B, C, H, W, K, unc_lo, unc_hi, unc_w);
    const Layout L = layout(a);
    VD3D_REQUIRE((size_t)workspace_bytes >= L.total, "monoflex_loss_forward: workspace of %lld bytes, %zu needed", workspace_bytes, L.total);
    char* ws = static_cast<char*>(workspace);
    auto* hm_part = reinterpret_cast<double*>(ws + L.hm_part);
    auto* row_part = reinterpret_cast<double*>(ws + L.row_part);
    cudaStream_t st = (cudaStream_t)stream;
    hm_kernel<<<a.hm_blocks, kThreads, 0, st>>>(a.map[M_HM], a.hm_t, (long long)B * C * H * W, hm_part);
    VD3D_CHECK_LAUNCH("monoflex_loss hm");
    rows_kernel<<<B, kRowThreads, 0, st>>>(a, row_part);
    VD3D_CHECK_LAUNCH("monoflex_loss rows");
    combine_kernel<<<1, 32, 0, st>>>(hm_part, row_part, a, terms, total, reinterpret_cast<float*>(ws + L.factors));
    VD3D_CHECK_LAUNCH("monoflex_loss combine");
    return VD3D_OK;
}

extern "C" int vd3d_monoflex_loss_backward(const void* const* maps, const void* const* targets, int B, int C, int H, int W, int K,
                                           float unc_lo, float unc_hi, float unc_w, const void* workspace, const float* grad_terms,
                                           const float* grad_total, float* const* grads, void* stream) {
    const int rc = check_sizes("monoflex_loss_backward", B, C, H, W, K);
    if (rc != VD3D_OK) return rc;
    VD3D_REQUIRE(maps && targets && workspace && grads, "monoflex_loss_backward: null pointer");
    for (int i = 0; i < kMaps; ++i) VD3D_REQUIRE(maps[i] && grads[i], "monoflex_loss_backward: null map or gradient %d", i);
    for (int i = 0; i < kTargets; ++i) VD3D_REQUIRE(targets[i], "monoflex_loss_backward: null target %d", i);
    const Args a = make_args(maps, targets, B, C, H, W, K, unc_lo, unc_hi, unc_w);
    const Layout L = layout(a);
    const float* factors = reinterpret_cast<const float*>(static_cast<const char*>(workspace) + L.factors);
    backward_kernel<<<dim3(cdiv((long long)H * W, kThreads), B), kThreads, 0, (cudaStream_t)stream>>>(
        a, factors, grad_terms, grad_total, grads[M_HM], grads[M_BBOX2D], grads[M_HPS], grads[M_ROT], grads[M_DIM], grads[M_REG],
        grads[M_DEPTH], grads[M_DUNC], grads[M_CUNC]);
    VD3D_CHECK_LAUNCH("monoflex_loss backward");
    return VD3D_OK;
}
