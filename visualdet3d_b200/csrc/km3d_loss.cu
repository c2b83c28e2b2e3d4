// Training loss of the KM3D head (KM3DHead.loss, R/networks/heads/km3d_head.py:316-351, with _neg_loss / _RegWeightedL1Loss /
// _RegL1Loss / _RotLoss from km3d_head.py:61-130, compute_rot_loss from R/networks/utils/rtm3d_utils.py:9-49 and Position_loss /
// gen_position from rtm3d_utils.py:230-455) for sm_90a.
//
// Forward, three launches whatever B, K and the number of objects (no memset, no host synchronisation, graph-capturable):
//   hm       grid-stride over hm [B][C][H][W] and hm_hp [B][9][H][W] in one launch (the first blocks over hm, the rest over hm_hp), each
//            block leaving its map's partials (positive sum, negative sum, positive count)
//   rows     one block per image: one thread per object row (the maps read at ind in NCHW, no permuted copy) for the keypoint, rotation,
//            L1 and position terms, and all threads striding over the image's K*9 keypoint rows (hp_ind) for hp_offset_loss; the image's
//            partials reduced in a fixed order
//   combine  one warp: partials summed in a fixed order in float64, each heatmap's own num_pos == 0 choice, the eleven terms, the
//            weighted total and the per-term factors the backward scales by
// Backward, one launch: each block owns a tile of one image's pixels and writes every gradient map there in full -- the heatmap
// derivatives, and zeros plus, at a gathered pixel, the contributions of the image's object rows (ind) or keypoint rows (hp_ind) at that
// pixel, summed in row order.
//
// The position term solves each row's 16 keypoint equations by least squares (km3d_position.cuh, shared with the detector's decode) with
// no jitter (the reference adds randn * 1e-8 to A^T A), and differentiates through the solve: with M = A^T A, x = M^-1 A^T b, g = dL/dx,
// u = M^-1 g and r = b - A x, dL/db = A u and dL/dA[:, 2] = r u_2 - (A u) x_2 (only A's third column varies).  The box score is the 3-D
// IoU of each row's own (prediction, ground truth) pair, read like boxes_iou3d_gpu reads [x, y, z, h, w, l, ry]; it carries no gradient.
//
// The prob / coor weight (exp_rampup(epoch)) is an argument, so a captured CUDA graph holds one epoch's weight.  No float atomics
// anywhere, so two runs give the same bits.  A row whose ind or hp_ind lies outside [0, H*W) is never read; it makes every loss (and
// every factor, so every gradient) NaN.
#include <algorithm>

#include "common.cuh"
#include "km3d_position.cuh"
#include "loss_common.cuh"
#include "rotated_overlap.cuh"

using vd3d::cdiv;
using vd3d::hm_grad;
using vd3d::kHmRec;
using vd3d::log_sigmoid;
using vd3d::sigmoid;
using vd3d::sign0;
using vd3d::warp_sum;

namespace {

constexpr int kThreads = 256;
constexpr int kMaxRows = 128;          // object rows per image (K)
constexpr int kJoints = 9;             // keypoints per object (Position_loss hard-codes 9)
constexpr int kMaxKp = kMaxRows * kJoints;
constexpr int kRowThreads = kMaxRows;
constexpr int kHmBlocksMax = 4 * vd3d::kNumSMs;
// hm, hp, hm_hp, hp_offset, wh, off, dim, rot, prob, coor (the reference's weight_dict order), then box_score (no weight)
enum { TM_HM, TM_HP, TM_HMHP, TM_HPO, TM_WH, TM_OFF, TM_DIM, TM_ROT, TM_PROB, TM_COOR, TM_SCORE, kTerms };
__constant__ float kWeight[TM_PROB] = {1.f, 1.f, 1.f, 1.f, 0.1f, 1.f, 2.f, 0.2f};

// the nine head maps, in the order of the C ABI, and their channel counts
enum { M_HM, M_WH, M_HPS, M_ROT, M_DIM, M_PROB, M_REG, M_HMHP, M_HPOFF, kMaps };
__constant__ int kMapCh[kMaps] = {0, 2, 18, 8, 3, 1, 2, kJoints, 2};
// an object row's gradient: the six maps gathered at ind, channels back to back
constexpr int kGathCh = 34;
__constant__ int kGOff[kMaps] = {0, 0, 2, 20, 28, 31, 32, 0, 0};

// targets, in the order of the C ABI
enum { T_HM, T_HMHP, T_IND, T_REG_MASK, T_HPS, T_HPS_MASK, T_DEP, T_ROTBIN, T_ROTRES, T_WH, T_DIM, T_REG, T_HP_IND, T_HP_MASK, T_HP_OFF,
       T_LOC, T_ORI, T_P2, kTargets };

// per-image partial record of the rows pass
enum { R_HP, R_HPM, R_CE, R_RES1, R_N1, R_RES2, R_N2, R_NREG, R_WH, R_DIM, R_OFF, R_HPO, R_NHPM, R_COOR, R_PROB, R_SCORE, R_MASKN, R_BAD,
       kRec };
// factors [kFac] f32 written by combine: d term / d (summed element) of each denominator
enum { F_HM, F_HMHP, F_HP, F_CE, F_RES1, F_RES2, F_WH, F_OFF, F_DIM, F_HPO, F_POS, kFac };

struct Args {
    const float* map[kMaps];
    const float* hm_t;
    const float* hmhp_t;
    const long long* ind;
    const unsigned char* reg_mask;
    const float* hps_t;
    const unsigned char* hps_mask;
    const float* dep;
    const long long* rotbin;
    const float* rotres;
    const float* wh_t;
    const float* dim_t;
    const float* reg_t;
    const long long* hp_ind;
    const unsigned char* hp_mask;
    const float* hpoff_t;
    const float* loc;
    const float* ori;
    const float* P2;
    int B, C, H, W, K, hm_blocks, hmhp_blocks;
    float output_w, rampup;
};

// the nine gradient maps, passed by value
struct Grads {
    float* p[kMaps];
};

// scales of the backward: d loss / d (summed element) of each term, grad_output included
struct Scales {
    float hm, hmhp, hp, ce, res1, res2, wh, off, dim, hpo, prob, coor;
};

__device__ __forceinline__ float clampf(float x, float lo, float hi) { return fminf(fmaxf(x, lo), hi); }

__global__ void __launch_bounds__(kThreads) hm_kernel(Args a, double* __restrict__ hm_part, double* __restrict__ hmhp_part) {
    const long long hw = (long long)a.H * a.W;
    if ((int)blockIdx.x < a.hm_blocks)
        vd3d::hm_block_partial<kThreads>(a.map[M_HM], a.hm_t, a.B * a.C * hw, blockIdx.x, a.hm_blocks, hm_part);
    else
        vd3d::hm_block_partial<kThreads>(a.map[M_HMHP], a.hmhp_t, a.B * kJoints * hw, blockIdx.x - a.hm_blocks, a.hmhp_blocks, hmhp_part);
}

// the 3-D IoU of one [x, y, z, h, w, l, ry] pair as boxes_iou3d_gpu computes it (R/lib/ops/iou3d/iou3d.py:37-71)
__device__ float iou3d_pair(const float* p, const float* q) {
    float bp[5], bq[5];
    const float* bx[2] = {p, q};
    float* bev[2] = {bp, bq};
    for (int i = 0; i < 2; ++i) {
        const float* s = bx[i];
        const float hl = s[5] / 2, hw = s[4] / 2;
        bev[i][0] = s[0] - hl; bev[i][1] = s[2] - hw; bev[i][2] = s[0] + hl; bev[i][3] = s[2] + hw; bev[i][4] = s[6];
    }
    const float ov = vd3d::rotated_overlap(bp, bq);
    const float lo = fmaxf(p[1] - p[3], q[1] - q[3]), hi = fminf(p[1], q[1]);
    const float oh = fmaxf(hi - lo, 0.f);
    const float o3 = ov * oh;
    const float va = p[3] * p[4] * p[5], vb = q[3] * q[4] * q[5];
    return o3 / fmaxf(va + vb - o3, 1e-7f);
}

// ---- one object row: its loss terms (rec, forward) or its gradient at the gathered pixel (g[kGathCh], backward) ----------------------
template <bool kGrad>
__device__ void row_eval(const Args& a, int b, int k, const Scales* s, float* rec, float* g) {
    const int HW = a.H * a.W;
    const size_t r = (size_t)b * a.K + k;
    const long long id = a.ind[r];
    if (id < 0 || id >= HW) {
        if (!kGrad) rec[R_BAD] = 1.f;
        return;
    }
    auto at = [&](int m, int c) { return a.map[m][((size_t)b * kMapCh[m] + c) * HW + id]; };
    if (kGrad)
        for (int c = 0; c < kGathCh; ++c) g[c] = 0.f;

    // hp_loss: every row, under hps_mask; dep transformed on a copy (the reference rewrites annotations['dep'] in place)
    {
        float l, ms;
        vd3d::weighted_l1_row<18, kGrad>([&](int c) { return at(M_HPS, c); }, a.hps_mask + r * 18, a.hps_t + r * 18, a.dep[r],
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
    // wh_loss, dim_loss, off_loss: L1 of the rows with reg_mask set (the others add 0 and get 0)
    if (valid) {
        const int ms[3] = {M_WH, M_DIM, M_REG};
        const float* ts[3] = {a.wh_t + r * 2, a.dim_t + r * 3, a.reg_t + r * 2};
        const int rs[3] = {R_WH, R_DIM, R_OFF};
        const float sc[3] = {kGrad ? s->wh : 0.f, kGrad ? s->dim : 0.f, kGrad ? s->off : 0.f};
        for (int i = 0; i < 3; ++i) {
            float l = 0.f;
            for (int c = 0; c < kMapCh[ms[i]]; ++c) {
                const float d = at(ms[i], c) - ts[i][c];
                l += fabsf(d);
                if (kGrad) g[kGOff[ms[i]] + c] += sign0(d) * sc[i];
            }
            if (!kGrad) rec[rs[i]] = l;
        }
        if (!kGrad) rec[R_NREG] = 1.f;
    }

    // ---- Position_loss: every row; counted where sum(hps_mask) > 15 ----
    const float ow = a.output_w;
    const float cy = truncf((float)id / ow);
    const float cx = (float)(int)fmod((double)id, (double)ow);
    float kx[kJoints], ky[kJoints], rot[8];
    for (int j = 0; j < kJoints; ++j) {
        kx[j] = (at(M_HPS, 2 * j) + cx) * 4.f;
        ky[j] = (at(M_HPS, 2 * j + 1) + cy) * 4.f;
    }
    for (int c = 0; c < 8; ++c) rot[c] = at(M_ROT, c);             // detached
    const float dw = at(M_DIM, 0), dh = at(M_DIM, 1), dl = at(M_DIM, 2);
    const float* P = a.P2 + (size_t)b * 12;
    vd3d::Km3dPosition gp;
    vd3d::km3d_gen_position(kx, ky, dw, dh, dl, rot, P, gp);
    float msum = 0.f;
    for (int c = 0; c < 18; ++c) msum += (float)a.hps_mask[r * 18 + c];
    const float lm = msum > 15.f ? 1.f : 0.f;
    const float* loc = a.loc + r * 3;
    const float dx = gp.pos[0] - loc[0], dy = gp.pos[1] - loc[1], dz = gp.pos[2] - loc[2];
    const float nrm = sqrtf(dx * dx + dy * dy + dz * dz);
    // the box score: IoU of (pos, clamp(dim, 0, 10), rot_y) with (location, dim_gt zeroed where dim < 0, ori); 0 for a negative dim
    const bool neg_dim = dw < 0.f || dh < 0.f || dl < 0.f;
    const float dmask = neg_dim ? 0.f : 1.f;
    float score;
    {
        const float* dt = a.dim_t + r * 3;
        const float pb[7] = {gp.pos[0], gp.pos[1], gp.pos[2], clampf(dw, 0.f, 10.f), clampf(dh, 0.f, 10.f), clampf(dl, 0.f, 10.f), gp.rot_y};
        const float qb[7] = {loc[0], loc[1], loc[2], dw < 0.f ? 0.f : dt[0], dh < 0.f ? 0.f : dt[1], dl < 0.f ? 0.f : dt[2], a.ori[r]};
        score = iou3d_pair(pb, qb) * lm * dmask;
    }
    const float xp = at(M_PROB, 0);
    if (!kGrad) {
        rec[R_COOR] = nrm * lm;
        rec[R_MASKN] = lm;
        rec[R_PROB] = ((1.f - score) * xp - log_sigmoid(xp)) * lm * dmask;
        rec[R_SCORE] = score * lm;
        return;
    }
    g[kGOff[M_PROB]] += (sigmoid(xp) - score) * lm * dmask * s->prob;
    if (!(lm != 0.f && nrm > 0.f)) return;
    // x: the solution before the offset, re-solved in float64 (no float32 rounding of pinv @ A^T or of the products with b), so the
    // direction (pos - location) / |pos - location| the gradient follows is the exact one even where the distance is a few cm
    double x[3], u[3];
    {
        double atb0 = 0.0, atb1 = 0.0, atb2 = 0.0;
        for (int q = 0; q < 16; ++q) {
            if (q & 1) atb1 -= gp.bv[q]; else atb0 -= gp.bv[q];
            atb2 += (double)gp.a2[q] * gp.bv[q];
        }
        for (int i = 0; i < 3; ++i) x[i] = gp.inv[i][0] * atb0 + gp.inv[i][1] * atb1 + gp.inv[i][2] * atb2;
    }
    const double ddx = x[0] - (double)P[3] / (double)P[0] - loc[0], ddy = x[1] - loc[1], ddz = x[2] - loc[2];
    const double dn = sqrt(ddx * ddx + ddy * ddy + ddz * ddz);
    if (!(dn > 0.0)) return;
    // d coor / d x
    const double gc = (double)s->coor * lm / dn;
    const double gx[3] = {gc * ddx, gc * ddy, gc * ddz};
    for (int i = 0; i < 3; ++i) u[i] = gp.inv[i][0] * gx[0] + gp.inv[i][1] * gx[1] + gp.inv[i][2] * gx[2];
    double gb[16], ga[16];
    for (int q = 0; q < 16; ++q) {
        const double a2 = gp.a2[q];
        const double au = ((q & 1) ? -u[1] : -u[0]) + a2 * u[2];
        const double res = (double)gp.bv[q] - (((q & 1) ? -x[1] : -x[0]) + a2 * x[2]);
        gb[q] = au;
        ga[q] = res * u[2] - au * x[2];
    }
    // b = B - a2 * C: into the keypoints (a2), B and C
    const float f = P[0];
    double g_lc = 0.0, g_wsn = 0.0, g_hh = 0.0, g_ls = 0.0, g_wc = 0.0;
    constexpr float kSxl[8] = {-1, -1, -1, 1, 1, 1, 1, -1}, kSxw[8] = {-1, 1, 1, 1, 1, -1, -1, -1}, kSy[8] = {-1, -1, 1, 1, -1, -1, 1, 1};
    constexpr float kScl[8] = {1, 1, 1, -1, -1, -1, -1, 1}, kScw[8] = {-1, 1, 1, 1, 1, -1, -1, -1};
    for (int j = 0; j < 8; ++j) {
        const double gnx = ga[2 * j] - gb[2 * j] * gp.cc[j], gny = ga[2 * j + 1] - gb[2 * j + 1] * gp.cc[j];
        const double gcc = -(gb[2 * j] * gp.a2[2 * j] + gb[2 * j + 1] * gp.a2[2 * j + 1]);
        g[kGOff[M_HPS] + 2 * j] += (float)(gnx * 4.0 / f);
        g[kGOff[M_HPS] + 2 * j + 1] += (float)(gny * 4.0 / f);
        g_lc += kSxl[j] * gb[2 * j];
        g_wsn += kSxw[j] * gb[2 * j];
        g_hh += kSy[j] * gb[2 * j + 1];
        g_ls += kScl[j] * gcc;
        g_wc += kScw[j] * gcc;
    }
    g[kGOff[M_DIM] + 0] += (float)(0.5 * (gp.co * g_wc + gp.si * g_wsn));
    g[kGOff[M_DIM] + 1] += (float)(0.5 * g_hh);
    g[kGOff[M_DIM] + 2] += (float)(0.5 * (gp.co * g_lc + gp.si * g_ls));
    // rot_y = alpha + atan2(kx8 - P[0,2], f): into the x of keypoint 8 (alpha comes from the detached rot)
    const double g_co = 0.5 * ((double)dl * g_lc + (double)dw * g_wc), g_si = 0.5 * ((double)dl * g_ls + (double)dw * g_wsn);
    const double g_ry = -(double)gp.si * g_co + (double)gp.co * g_si;
    const double y8 = (double)kx[8] - (double)P[2];
    g[kGOff[M_HPS] + 16] += (float)(g_ry * (double)f / (y8 * y8 + (double)f * f) * 4.0);
}

// Args from the C ABI's pointer arrays
Args make_args(const void* const* maps, const void* const* targets, int B, int C, int H, int W, int K, float output_w, float rampup) {
    Args a;
    for (int m = 0; m < kMaps; ++m) a.map[m] = static_cast<const float*>(maps[m]);
    a.hm_t = static_cast<const float*>(targets[T_HM]);
    a.hmhp_t = static_cast<const float*>(targets[T_HMHP]);
    a.ind = static_cast<const long long*>(targets[T_IND]);
    a.reg_mask = static_cast<const unsigned char*>(targets[T_REG_MASK]);
    a.hps_t = static_cast<const float*>(targets[T_HPS]);
    a.hps_mask = static_cast<const unsigned char*>(targets[T_HPS_MASK]);
    a.dep = static_cast<const float*>(targets[T_DEP]);
    a.rotbin = static_cast<const long long*>(targets[T_ROTBIN]);
    a.rotres = static_cast<const float*>(targets[T_ROTRES]);
    a.wh_t = static_cast<const float*>(targets[T_WH]);
    a.dim_t = static_cast<const float*>(targets[T_DIM]);
    a.reg_t = static_cast<const float*>(targets[T_REG]);
    a.hp_ind = static_cast<const long long*>(targets[T_HP_IND]);
    a.hp_mask = static_cast<const unsigned char*>(targets[T_HP_MASK]);
    a.hpoff_t = static_cast<const float*>(targets[T_HP_OFF]);
    a.loc = static_cast<const float*>(targets[T_LOC]);
    a.ori = static_cast<const float*>(targets[T_ORI]);
    a.P2 = static_cast<const float*>(targets[T_P2]);
    a.B = B; a.C = C; a.H = H; a.W = W; a.K = K;
    const long long hw = (long long)H * W;
    a.hm_blocks = (int)std::min<long long>(cdiv((long long)B * C * hw, kThreads * 8), kHmBlocksMax);
    a.hmhp_blocks = (int)std::min<long long>(cdiv((long long)B * kJoints * hw, kThreads * 8), kHmBlocksMax);
    a.output_w = output_w; a.rampup = rampup;
    return a;
}

// one keypoint row (hp_ind) of hp_offset_loss: returns false for an hp_ind outside [0, H*W); l / ms: its L1 and mask; gd: d l / d map
__device__ __forceinline__ bool kp_row(const Args& a, int b, int j, float* l, float* ms, float* gd, float scale) {
    const int HW = a.H * a.W;
    const size_t r = (size_t)b * a.K * kJoints + j;
    const long long id = a.hp_ind[r];
    if (id < 0 || id >= HW) return false;
    const float m = (float)a.hp_mask[r];
    float s = 0.f;
    for (int c = 0; c < 2; ++c) {
        const float d = a.map[M_HPOFF][((size_t)b * 2 + c) * HW + id] * m - a.hpoff_t[r * 2 + c] * m;
        s += fabsf(d);
        if (gd) gd[c] = sign0(d) * m * scale;
    }
    if (l) { *l = s; *ms = m; }
    return true;
}

// ---- the rows pass: one block per image ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kRowThreads) rows_kernel(Args a, double* __restrict__ partial) {
    __shared__ double s_red[kRowThreads / 32][kRec];
    const int b = blockIdx.x, k = threadIdx.x;
    float rec[kRec];
#pragma unroll
    for (int i = 0; i < kRec; ++i) rec[i] = 0.f;
    if (k < a.K) row_eval<false>(a, b, k, nullptr, rec, nullptr);
    for (int j = k; j < a.K * kJoints; j += kRowThreads) {
        float l, ms;
        if (kp_row(a, b, j, &l, &ms, nullptr, 0.f)) {
            rec[R_HPO] += l;
            rec[R_NHPM] += ms;
        } else {
            rec[R_BAD] = 1.f;
        }
    }
    const double v = vd3d::block_partial<kRowThreads, kRec>(rec, s_red);
    if (threadIdx.x < kRec) partial[(size_t)b * kRec + threadIdx.x] = v;
}

// ---- combine: one warp; sums in a fixed order (vd3d::warp_sum: lane-strided, then a shuffle tree) -----------------------------

// _neg_loss from its summed partials: the term and its factor (the num_pos == 0 choice made here)
__device__ __forceinline__ float focal_term(const double* hv, float& factor) {
    const float pos = (float)hv[0], neg = (float)hv[1], npos = (float)hv[2];
    factor = npos == 0.f ? -1.f : -1.f / npos;
    return npos == 0.f ? -neg : -(pos + neg) / npos;
}

__global__ void combine_kernel(const double* __restrict__ hm_part, const double* __restrict__ hmhp_part, const double* __restrict__ row_part,
                               Args a, float* __restrict__ terms, float* __restrict__ total, float* __restrict__ factors) {
    const int lane = threadIdx.x;
    double hmv[kHmRec], hpv[kHmRec], rv[kRec];
    for (int i = 0; i < kHmRec; ++i) hmv[i] = warp_sum(hm_part + i, a.hm_blocks, kHmRec, lane);
    for (int i = 0; i < kHmRec; ++i) hpv[i] = warp_sum(hmhp_part + i, a.hmhp_blocks, kHmRec, lane);
    for (int i = 0; i < kRec; ++i) rv[i] = warp_sum(row_part + i, a.B, kRec, lane);
    if (lane != 0) return;
    float t[kTerms], f[kFac];
    t[TM_HM] = focal_term(hmv, f[F_HM]);
    t[TM_HMHP] = focal_term(hpv, f[F_HMHP]);
    const float hp_den = (float)rv[R_HPM] + 1e-4f;
    t[TM_HP] = (float)rv[R_HP] / hp_den;
    f[F_HP] = 1.f / hp_den;
    const float nreg = (float)rv[R_NREG];
    const float wh_den = nreg * 2.f + 1e-4f, dim_den = nreg * 3.f + 1e-4f, hpo_den = (float)rv[R_NHPM] * 2.f + 1e-4f;
    t[TM_WH] = (float)rv[R_WH] / wh_den;
    t[TM_OFF] = (float)rv[R_OFF] / wh_den;
    t[TM_DIM] = (float)rv[R_DIM] / dim_den;
    t[TM_HPO] = (float)rv[R_HPO] / hpo_den;
    f[F_WH] = f[F_OFF] = 1.f / wh_den;
    f[F_DIM] = 1.f / dim_den;
    f[F_HPO] = 1.f / hpo_den;
    const float rows = (float)((long long)a.B * a.K);
    float rot = (float)rv[R_CE] / rows;
    f[F_CE] = 1.f / rows;
    f[F_RES1] = rv[R_N1] > 0 ? 1.f / (float)rv[R_N1] : 0.f;
    f[F_RES2] = rv[R_N2] > 0 ? 1.f / (float)rv[R_N2] : 0.f;
    if (rv[R_N1] > 0) rot += (float)rv[R_RES1] / (float)rv[R_N1];
    if (rv[R_N2] > 0) rot += (float)rv[R_RES2] / (float)rv[R_N2];
    t[TM_ROT] = rot;
    const float maskn = (float)rv[R_MASKN];
    t[TM_PROB] = (float)rv[R_PROB] / (maskn + 1.f);
    t[TM_COOR] = (float)rv[R_COOR] / (maskn + 1.f);
    t[TM_SCORE] = (float)rv[R_SCORE] / (maskn + 1e-3f);
    f[F_POS] = 1.f / (maskn + 1.f);
    const bool bad = rv[R_BAD] > 0;
    float sum = 0.f;
    for (int i = 0; i < kTerms; ++i) {
        if (bad) t[i] = __int_as_float(0x7fc00000);
        terms[i] = t[i];
        if (i < TM_SCORE) sum = sum + t[i] * (i < TM_PROB ? kWeight[i] : a.rampup);
    }
    *total = sum;
    for (int i = 0; i < kFac; ++i) factors[i] = bad ? __int_as_float(0x7fc00000) : f[i];
}

// ---- backward ---------------------------------------------------------------------------------------------------------------------
// compacts, in index order, the entries i < n of idx (one image's ind or hp_ind) that fall in the tile [p0, p0 + kThreads)
__device__ int compact_tile(const long long* idx, int n, int p0, int HW, int* s_row, int* s_pix, int* s_cnt) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int total = 0;
    for (int base = 0; base < n; base += kThreads) {
        const int i = base + threadIdx.x;
        long long id = -1;
        bool hit = false;
        if (i < n) {
            id = idx[i];
            hit = id >= p0 && id < p0 + kThreads && id < HW;
        }
        const unsigned bal = __ballot_sync(0xffffffffu, hit);
        if (lane == 0) s_cnt[warp] = __popc(bal);
        __syncthreads();
        int off = 0, nm = 0;
        for (int w = 0; w < kThreads / 32; ++w) {
            if (w < warp) off += s_cnt[w];
            nm += s_cnt[w];
        }
        if (hit) {
            const int slot = total + off + __popc(bal & ((1u << lane) - 1u));
            s_row[slot] = i;
            s_pix[slot] = (int)id;
        }
        total += nm;
        __syncthreads();
    }
    return total;
}

__global__ void __launch_bounds__(kThreads) backward_kernel(Args a, const float* __restrict__ factors, const float* __restrict__ g_terms,
                                                            const float* __restrict__ g_total, Grads g) {
    __shared__ int s_row[kMaxRows], s_pix[kMaxRows];
    __shared__ int s_krow[kMaxKp], s_kpix[kMaxKp];
    __shared__ int s_cnt[kThreads / 32];
    __shared__ float s_g[kMaxRows][kGathCh];
    __shared__ float s_kg[kMaxKp][2];
    const int b = blockIdx.y, HW = a.H * a.W;
    const int p0 = blockIdx.x * kThreads;
    // the image's object rows and keypoint rows whose pixel falls in this tile, compacted in row order
    const int nm = compact_tile(a.ind + (size_t)b * a.K, a.K, p0, HW, s_row, s_pix, s_cnt);
    const int nk = compact_tile(a.hp_ind + (size_t)b * a.K * kJoints, a.K * kJoints, p0, HW, s_krow, s_kpix, s_cnt);
    Scales s;
    {
        float gt[kTerms];
        const float gtot = g_total ? *g_total : 0.f;
        for (int i = 0; i < kTerms; ++i) {
            const float w = i < TM_PROB ? kWeight[i] : (i < TM_SCORE ? a.rampup : 0.f);
            gt[i] = (g_terms ? g_terms[i] : 0.f) + w * gtot;
        }
        s.hm = factors[F_HM] * gt[TM_HM];
        s.hmhp = factors[F_HMHP] * gt[TM_HMHP];
        s.hp = factors[F_HP] * gt[TM_HP];
        s.hpo = factors[F_HPO] * gt[TM_HPO];
        s.wh = factors[F_WH] * gt[TM_WH];
        s.off = factors[F_OFF] * gt[TM_OFF];
        s.dim = factors[F_DIM] * gt[TM_DIM];
        s.ce = factors[F_CE] * gt[TM_ROT];
        s.res1 = factors[F_RES1] * gt[TM_ROT];
        s.res2 = factors[F_RES2] * gt[TM_ROT];
        s.prob = factors[F_POS] * gt[TM_PROB];
        s.coor = factors[F_POS] * gt[TM_COOR];
    }
    if (threadIdx.x < nm) row_eval<true>(a, b, s_row[threadIdx.x], &s, nullptr, s_g[threadIdx.x]);
    for (int i = threadIdx.x; i < nk; i += kThreads) kp_row(a, b, s_krow[i], nullptr, nullptr, s_kg[i], s.hpo);
    __syncthreads();
    const int p = p0 + threadIdx.x;
    if (p >= HW) return;
    for (int m = M_WH; m <= M_REG; ++m) {
        for (int c = 0; c < kMapCh[m]; ++c) {
            float v = 0.f;
            for (int i = 0; i < nm; ++i)
                if (s_pix[i] == p) v += s_g[i][kGOff[m] + c];
            g.p[m][((size_t)b * kMapCh[m] + c) * HW + p] = v;
        }
    }
    for (int c = 0; c < 2; ++c) {
        float v = 0.f;
        for (int i = 0; i < nk; ++i)
            if (s_kpix[i] == p) v += s_kg[i][c];
        g.p[M_HPOFF][((size_t)b * 2 + c) * HW + p] = v;
    }
    for (int c = 0; c < a.C; ++c) {
        const size_t i = ((size_t)b * a.C + c) * HW + p;
        g.p[M_HM][i] = hm_grad(a.map[M_HM][i], a.hm_t[i]) * s.hm;
    }
    for (int c = 0; c < kJoints; ++c) {
        const size_t i = ((size_t)b * kJoints + c) * HW + p;
        g.p[M_HMHP][i] = hm_grad(a.map[M_HMHP][i], a.hmhp_t[i]) * s.hmhp;
    }
}

struct Layout {
    size_t hm_part, hmhp_part, row_part, factors, total;
};

Layout layout(const Args& a) {
    auto up = [](size_t x) { return (x + 255) & ~(size_t)255; };
    Layout L;
    L.hm_part = 0;
    L.hmhp_part = up((size_t)a.hm_blocks * kHmRec * sizeof(double));
    L.row_part = L.hmhp_part + up((size_t)a.hmhp_blocks * kHmRec * sizeof(double));
    L.factors = L.row_part + up((size_t)a.B * kRec * sizeof(double));
    L.total = L.factors + kFac * sizeof(float);
    return L;
}

int check_sizes(const char* who, int B, int C, int H, int W, int K, float output_w) {
    VD3D_REQUIRE(B > 0 && C > 0 && H > 0 && W > 0 && K > 0 && K <= kMaxRows, "%s: bad sizes B=%d C=%d H=%d W=%d K=%d (1 <= K <= %d)", who, B,
                 C, H, W, K, kMaxRows);
    VD3D_REQUIRE((long long)H * W < (1ll << 31), "%s: H*W = %lld pixels, at most 2^31 - 1 supported", who, (long long)H * W);
    VD3D_REQUIRE(output_w > 0.f, "%s: output_w must be > 0, got %g", who, output_w);
    return VD3D_OK;
}

}  // namespace

extern "C" long long vd3d_km3d_loss_workspace_bytes(int B, int C, int H, int W, int K) {
    const int rc = check_sizes("km3d_loss_workspace_bytes", B, C, H, W, K, 1.f);
    if (rc != VD3D_OK) return rc;
    const void* none[kTargets] = {};
    return (long long)layout(make_args(none, none, B, C, H, W, K, 1.f, 0.f)).total;
}

extern "C" int vd3d_km3d_loss_forward(const void* const* maps, const void* const* targets, int B, int C, int H, int W, int K, float output_w,
                                      float rampup, void* workspace, long long workspace_bytes, float* terms, float* total, void* stream) {
    const int rc = check_sizes("km3d_loss_forward", B, C, H, W, K, output_w);
    if (rc != VD3D_OK) return rc;
    VD3D_REQUIRE(maps && targets && workspace && terms && total, "km3d_loss_forward: null pointer");
    for (int i = 0; i < kMaps; ++i) VD3D_REQUIRE(maps[i], "km3d_loss_forward: null map %d", i);
    for (int i = 0; i < kTargets; ++i) VD3D_REQUIRE(targets[i], "km3d_loss_forward: null target %d", i);
    const Args a = make_args(maps, targets, B, C, H, W, K, output_w, rampup);
    const Layout L = layout(a);
    VD3D_REQUIRE((size_t)workspace_bytes >= L.total, "km3d_loss_forward: workspace of %lld bytes, %zu needed", workspace_bytes, L.total);
    char* ws = static_cast<char*>(workspace);
    auto* hm_part = reinterpret_cast<double*>(ws + L.hm_part);
    auto* hmhp_part = reinterpret_cast<double*>(ws + L.hmhp_part);
    auto* row_part = reinterpret_cast<double*>(ws + L.row_part);
    cudaStream_t st = (cudaStream_t)stream;
    hm_kernel<<<a.hm_blocks + a.hmhp_blocks, kThreads, 0, st>>>(a, hm_part, hmhp_part);
    VD3D_CHECK_LAUNCH("km3d_loss hm");
    rows_kernel<<<B, kRowThreads, 0, st>>>(a, row_part);
    VD3D_CHECK_LAUNCH("km3d_loss rows");
    combine_kernel<<<1, 32, 0, st>>>(hm_part, hmhp_part, row_part, a, terms, total, reinterpret_cast<float*>(ws + L.factors));
    VD3D_CHECK_LAUNCH("km3d_loss combine");
    return VD3D_OK;
}

extern "C" int vd3d_km3d_loss_backward(const void* const* maps, const void* const* targets, int B, int C, int H, int W, int K,
                                       float output_w, float rampup, const void* workspace, const float* grad_terms, const float* grad_total,
                                       float* const* grads, void* stream) {
    const int rc = check_sizes("km3d_loss_backward", B, C, H, W, K, output_w);
    if (rc != VD3D_OK) return rc;
    VD3D_REQUIRE(maps && targets && workspace && grads, "km3d_loss_backward: null pointer");
    for (int i = 0; i < kMaps; ++i) VD3D_REQUIRE(maps[i] && grads[i], "km3d_loss_backward: null map or gradient %d", i);
    for (int i = 0; i < kTargets; ++i) VD3D_REQUIRE(targets[i], "km3d_loss_backward: null target %d", i);
    const Args a = make_args(maps, targets, B, C, H, W, K, output_w, rampup);
    const Layout L = layout(a);
    const float* factors = reinterpret_cast<const float*>(static_cast<const char*>(workspace) + L.factors);
    Grads o;
    for (int i = 0; i < kMaps; ++i) o.p[i] = grads[i];
    backward_kernel<<<dim3(cdiv((long long)H * W, kThreads), B), kThreads, 0, (cudaStream_t)stream>>>(a, factors, grad_terms, grad_total, o);
    VD3D_CHECK_LAUNCH("km3d_loss backward");
    return VD3D_OK;
}
