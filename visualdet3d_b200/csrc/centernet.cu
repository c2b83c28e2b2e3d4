// CenterNet-style decode for the MonoFlex head (MonoFlexHead.get_bboxes, R/heads/monoflex_head.py:114-179), batched and
// fully on the device: sigmoid + 3x3 local-maximum test (`_nms`, R/utils/rtm3d_utils.py:122-127), top-K over (class, y, x)
// (`_topk`, :201-216), gather of the 8 regression maps at the K peaks (`_gather_output`, monoflex_head.py:45-75), depth from
// exp(-d) and from three keypoint-height groups (`decode_depth_from_keypoints`, rtm3d_utils.py:141-182) merged by inverse
// uncertainty (`merge_depth`, :86-91), alpha from the two-bin rotation (`_decode_alpha`, :106-112), x4 up-scaling, ClipBoxes
// and class-agnostic torchvision-style NMS.
//
// Order equivalence: the reference keeps the K best peaks, then drops scores <= score_thr; selecting peaks > score_thr first
// and keeping the best K of those yields the same set and order (scores are sorted descending, ties by flat index).
#include "decode_common.cuh"
#include "km3d_position.cuh"

namespace vd3d {

struct CnLayout {            // channel offsets inside the concatenated head-output tensor [B][H][W][cs]
    int cs, hm, bbox2d, hps, rot, dim, reg, depth, dunc, cunc;
};

// ---- stage 1: peaks (3x3 local maxima) of channels base .. base + nch - 1 above thr -> unordered key lists ----------------------------
// per_channel: one list per (image, channel) with index y * W + x (KM3D's keypoint joints); otherwise one list per image with the flat
// index (c * H + y) * W + x.
__global__ void cn_peaks_kernel(const float* __restrict__ out, int B, int H, int W, int cs, int base, int nch, bool per_channel, float thr,
                                int cap, unsigned long long* __restrict__ keys, int* __restrict__ ncand) {
    long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    long long total = (long long)B * nch * H * W;
    if (idx >= total) return;
    int w = (int)(idx % W); long long r = idx / W; int h = (int)(r % H); r /= H; int c = (int)(r % nch); int b = (int)(r / nch);
    const float* p = out + ((long long)b * H * W) * cs + base + c;
    float s = sigmoid_ref(__ldg(p + ((long long)h * W + w) * cs));
    if (!(s > thr)) return;
    float m = s;
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
        for (int dx = -1; dx <= 1; ++dx) {
            int hh = h + dy, ww = w + dx;
            if ((dy | dx) == 0 || hh < 0 || hh >= H || ww < 0 || ww >= W) continue;
            m = fmaxf(m, sigmoid_ref(__ldg(p + ((long long)hh * W + ww) * cs)));
        }
    if (m != s) return;                                  // keep = (hmax == heat)
    const int list = per_channel ? b * nch + c : b;
    int slot = atomicAdd(ncand + list, 1);
    if (slot >= cap) return;
    keys[(long long)list * cap + slot] = score_key(s, (unsigned int)((per_channel ? h : c * H + h) * W + w));
}

// ---- stage 2: one CTA per image: sort, keep K, decode, NMS ----------------------------------------------------------------
constexpr int CN_THREADS = 1024;
constexpr int CN_MAXK = 128;
constexpr int CN_MASK_WPR = CN_MAXK / 64;      // words per row of the NMS sweep's suppression mask

__global__ void __launch_bounds__(CN_THREADS) cn_decode_nms_kernel(
    const float* __restrict__ out, const float* __restrict__ P2, int H, int W, int ncls, CnLayout L, int cap, int cap_pow2, int K,
    float unc_lo, float unc_hi, double iou_thr, float img_w, float img_h, int out_cap,
    const unsigned long long* __restrict__ keys, const int* __restrict__ ncand,
    float* __restrict__ o_scores, float* __restrict__ o_boxes, long long* __restrict__ o_cls, int* __restrict__ o_index,
    int* __restrict__ o_count, int* __restrict__ o_ncand) {
    extern __shared__ __align__(16) unsigned char sm_raw[];
    unsigned long long* skey = reinterpret_cast<unsigned long long*>(sm_raw);            // [cap_pow2]
    __shared__ float sbox[CN_MAXK][11];
    __shared__ float4 sbox4[CN_MAXK];
    __shared__ float sarea[CN_MAXK];
    __shared__ int skeep[CN_MAXK];
    __shared__ unsigned long long smask[64 * CN_MASK_WPR];
    const int b = blockIdx.x, t = threadIdx.x;
    int n = ncand[b];
    if (t == 0) o_ncand[b] = n;
    if (n > cap) { if (t == 0) o_count[b] = -1; return; }
    cap_pow2 = min(next_pow2(n, 2), cap_pow2);          // sort only the occupied power of two (block-uniform)
    for (int i = t; i < cap_pow2; i += CN_THREADS) skey[i] = (i < n) ? keys[(long long)b * cap + i] : ~0ull;
    __syncthreads();
    block_sort<CN_THREADS, false>(skey, nullptr, cap_pow2);
    const int nk = min(n, K);
    if (t < nk) {
        unsigned int flat = key_index(skey[t]);
        int x = flat % W; int r = flat / W; int y = r % H;
        const float* px = out + (((long long)b * H + y) * W + x) * L.cs;
        float xs = (float)x, ys = (float)y;
        float bx1 = xs - px[L.bbox2d + 0], by1 = ys - px[L.bbox2d + 1], bx2 = xs + px[L.bbox2d + 2], by2 = ys + px[L.bbox2d + 3];
        // depths
        float d0 = expf(-px[L.depth]);
        const float* kp = px + L.hps;                        // [10][2]
        float ph = px[L.dim + 1];
        float f = P2[12 * b + 0];
        float fh = f * ph;
        const float EPS = 1e-8f;
        float ch = kp[2 * 8 + 1] - kp[2 * 9 + 1];
        float h02a = kp[2 * 7 + 1] - kp[2 * 0 + 1], h02b = kp[2 * 3 + 1] - kp[2 * 4 + 1];
        float h13a = kp[2 * 2 + 1] - kp[2 * 1 + 1], h13b = kp[2 * 6 + 1] - kp[2 * 5 + 1];
        float dc = fh / (fmaxf(ch, 0.f) * 4.f + EPS);
        float d02 = (fh / (fmaxf(h02a, 0.f) * 4.f + EPS) + fh / (fmaxf(h02b, 0.f) * 4.f + EPS)) / 2.f;
        float d13 = (fh / (fmaxf(h13a, 0.f) * 4.f + EPS) + fh / (fmaxf(h13b, 0.f) * 4.f + EPS)) / 2.f;
        dc = fminf(fmaxf(dc, 0.1f), 100.f); d02 = fminf(fmaxf(d02, 0.1f), 100.f); d13 = fminf(fmaxf(d13, 0.1f), 100.f);
        float u0 = expf(fminf(fmaxf(px[L.dunc], unc_lo), unc_hi));
        float u1 = expf(fminf(fmaxf(px[L.cunc + 0], unc_lo), unc_hi));
        float u2 = expf(fminf(fmaxf(px[L.cunc + 1], unc_lo), unc_hi));
        float u3 = expf(fminf(fmaxf(px[L.cunc + 2], unc_lo), unc_hi));
        float w0 = 1.f / u0, w1 = 1.f / u1, w2 = 1.f / u2, w3 = 1.f / u3;
        float ws = ((w0 + w1) + w2) + w3;
        w0 /= ws; w1 /= ws; w2 /= ws; w3 /= ws;
        float z = ((d0 * w0 + dc * w1) + d02 * w2) + d13 * w3;
        // alpha
        const float* rot = px + L.rot;
        float a1 = atanf(rot[2] / rot[3]) + (-0.5f * 3.14159265358979323846f);
        float a2 = atanf(rot[6] / rot[7]) + (0.5f * 3.14159265358979323846f);
        float sel = (rot[1] > rot[5]) ? 1.f : 0.f;
        float alpha = a1 * sel + a2 * (1.f - sel);
        float cx = (xs + px[L.reg + 0]) * 4.f, cy = (ys + px[L.reg + 1]) * 4.f;
        bx1 *= 4.f; by1 *= 4.f; bx2 *= 4.f; by2 *= 4.f;
        bx1 = fmaxf(bx1, 0.f); by1 = fmaxf(by1, 0.f); bx2 = fminf(bx2, img_w); by2 = fminf(by2, img_h);
        float* sb = sbox[t];
        sb[0] = bx1; sb[1] = by1; sb[2] = bx2; sb[3] = by2; sb[4] = cx; sb[5] = cy; sb[6] = z;
        sb[7] = px[L.dim + 0]; sb[8] = px[L.dim + 1]; sb[9] = px[L.dim + 2]; sb[10] = alpha;
        const float4 bx = make_float4(bx1, by1, bx2, by2);
        sbox4[t] = bx;
        sarea[t] = box_area(bx);
    }
    __syncthreads();
    const int nkeep = nms_sweep<CN_THREADS>(sbox4, sarea, nk, CN_MASK_WPR, iou_thr, smask, skeep);
    // ordered write-out of the kept rows, one per thread (nkeep <= K < CN_THREADS)
    if (t < nkeep) {
        const int k = t, i = skeep[k];
        const unsigned long long key = skey[i];
        const unsigned int flat = key_index(key);
        o_scores[(long long)b * out_cap + k] = key_score(key);
        o_index[(long long)b * out_cap + k] = (int)flat;
        o_cls[(long long)b * out_cap + k] = (long long)(flat / (unsigned int)(H * W));
        float* op = o_boxes + ((long long)b * out_cap + k) * 11;
#pragma unroll
        for (int q = 0; q < 11; ++q) op[q] = sbox[i][q];
    }
    if (t == 0) o_count[b] = nkeep;
}

// ================================================================================================================
// KM3D: KM3DHead.get_bboxes / _decode (R/heads/km3d_head.py:155-314) + gen_position (R/utils/rtm3d_utils.py:314-455)
// ================================================================================================================
struct KmLayout { int cs, hm, wh, hps, rot, dim, prob, reg, hm_hp, hp_offset; };

constexpr int KM_J = 9;

__global__ void __launch_bounds__(CN_THREADS) km3d_decode_nms_kernel(
    const float* __restrict__ out, const float* __restrict__ P2, int H, int W, int ncls, KmLayout L, int cap, int cap_pow2, int hp_cap,
    int hp_cap_pow2, int K, double iou_thr, float img_w, float img_h, int out_cap,
    const unsigned long long* __restrict__ keys, const int* __restrict__ ncand,
    const unsigned long long* __restrict__ hp_keys, const int* __restrict__ hp_ncand,
    float* __restrict__ o_scores, float* __restrict__ o_boxes, long long* __restrict__ o_cls, int* __restrict__ o_index,
    int* __restrict__ o_count, int* __restrict__ o_ncand) {
    extern __shared__ __align__(16) unsigned char sm_raw[];
    unsigned long long* skey = reinterpret_cast<unsigned long long*>(sm_raw);            // [max(cap_pow2, hp_cap_pow2)]
    __shared__ float hpx[KM_J][CN_MAXK], hpy[KM_J][CN_MAXK], hps_[KM_J][CN_MAXK];
    __shared__ int hpn[KM_J];
    __shared__ unsigned long long dkey[CN_MAXK];
    __shared__ float sbox[CN_MAXK][11];
    __shared__ float4 sbox4[CN_MAXK];
    __shared__ float sarea[CN_MAXK];
    __shared__ int skeep[CN_MAXK];
    __shared__ unsigned long long smask[64 * CN_MASK_WPR];
    const int b = blockIdx.x, t = threadIdx.x;
    int n = ncand[b];
    if (t == 0) o_ncand[b] = n;
    bool overflow = n > cap;
    for (int j = 0; j < KM_J; ++j) overflow = overflow || hp_ncand[b * KM_J + j] > hp_cap;
    if (overflow) { if (t == 0) o_count[b] = -1; return; }      // fixed-capacity candidate lists overflowed: reported, never silently truncated
    // ---- detection peaks: sort, keep the best K -----------------------------------------------------------------------------
    cap_pow2 = min(next_pow2(n, 2), cap_pow2);          // sort only the occupied power of two (block-uniform)
    for (int i = t; i < cap_pow2; i += CN_THREADS) skey[i] = (i < n) ? keys[(long long)b * cap + i] : ~0ull;
    __syncthreads();
    block_sort<CN_THREADS, false>(skey, nullptr, cap_pow2);
    const int nk = min(n, K);
    if (t < nk) dkey[t] = skey[t];
    __syncthreads();
    // ---- keypoint heat-map peaks per joint: best K of those above 0.1, with their sub-pixel offsets ---------------------------
    for (int j = 0; j < KM_J; ++j) {
        int nj = min(hp_ncand[b * KM_J + j], hp_cap);
        const int hp2 = min(next_pow2(nj, 2), hp_cap_pow2);
        __syncthreads();                                     // the previous joint's readers of skey are done
        for (int i = t; i < hp2; i += CN_THREADS) skey[i] = (i < nj) ? hp_keys[((long long)b * KM_J + j) * hp_cap + i] : ~0ull;
        __syncthreads();
        block_sort<CN_THREADS, false>(skey, nullptr, hp2);
        int m = min(nj, K);
        if (t < m) {
            unsigned long long key = skey[t];
            unsigned int flat = key_index(key);
            int x = flat % W, y = flat / W;
            const float* px = out + (((long long)b * H + y) * W + x) * L.cs;
            hpx[j][t] = (float)x + px[L.hp_offset + 0];
            hpy[j][t] = (float)y + px[L.hp_offset + 1];
            hps_[j][t] = key_score(key);
        }
        if (t == 0) hpn[j] = m;
        __syncthreads();
    }
    // ---- per detection decode --------------------------------------------------------------------------------------------------
    if (t < nk) {
        unsigned int flat = key_index(dkey[t]);
        int x = flat % W; int r = flat / W; int y = r % H;
        const float* px = out + (((long long)b * H + y) * W + x) * L.cs;
        float xs0 = (float)x, ys0 = (float)y;
        float kx[KM_J], ky[KM_J];
#pragma unroll
        for (int j = 0; j < KM_J; ++j) { kx[j] = px[L.hps + 2 * j] + xs0; ky[j] = px[L.hps + 2 * j + 1] + ys0; }
        float xs = xs0 + px[L.reg + 0], ys = ys0 + px[L.reg + 1];
        float bw = px[L.wh + 0], bh = px[L.wh + 1];
        float l = xs - bw / 2, tp = ys - bh / 2, rr = xs + bw / 2, bt = ys + bh / 2;
        // keypoint refinement with the heat-map peaks (km3d_head.py:195-241)
        const float gate = fmaxf(bt - tp, rr - l) * 0.3f;
#pragma unroll
        for (int j = 0; j < KM_J; ++j) {
            float best = 3.4e38f; int bi = -1;
            int m = hpn[j];
            for (int q = 0; q < K; ++q) {
                float qx = (q < m) ? hpx[j][q] : -10000.f, qy = (q < m) ? hpy[j][q] : -10000.f;   // masked peaks sit at (-10000, -10000)
                float dx = kx[j] - qx, dy = ky[j] - qy;
                float d = sqrtf(dx * dx + dy * dy);
                if (d < best) { best = d; bi = q; }
            }
            float qx = (bi < m) ? hpx[j][bi] : -10000.f, qy = (bi < m) ? hpy[j][bi] : -10000.f;
            float qs = (bi < m) ? hps_[j][bi] : -1.f;
            bool reject = (qx < l) || (qx > rr) || (qy < tp) || (qy > bt) || (qs < 0.1f) || (best > gate);
            if (!reject) { kx[j] = qx; ky[j] = qy; }
        }
#pragma unroll
        for (int j = 0; j < KM_J; ++j) { kx[j] *= 4.f; ky[j] *= 4.f; }
        l *= 4.f; tp *= 4.f; rr *= 4.f; bt *= 4.f;
        // gen_position
        const float* P = P2 + 12 * b;
        vd3d::Km3dPosition gp;
        const float dw = px[L.dim + 0], dh = px[L.dim + 1], dl = px[L.dim + 2];
        vd3d::km3d_gen_position(kx, ky, dw, dh, dl, px + L.rot, P, gp);
        const float alpha = gp.alpha;
        const float* pos = gp.pos;
        float z3 = pos[2];
        float cx3 = (pos[0] * P[0] + P[3] + P[2] * z3) / z3;
        float cy3 = (pos[1] * P[5] + P[7] + P[6] * z3) / z3;
        l = fmaxf(l, 0.f); tp = fmaxf(tp, 0.f); rr = fminf(rr, img_w); bt = fminf(bt, img_h);
        float* sb = sbox[t];
        sb[0] = l; sb[1] = tp; sb[2] = rr; sb[3] = bt; sb[4] = cx3; sb[5] = cy3; sb[6] = z3; sb[7] = dw; sb[8] = dh; sb[9] = dl; sb[10] = alpha;
        const float4 bx = make_float4(l, tp, rr, bt);
        sbox4[t] = bx;
        sarea[t] = box_area(bx);
    }
    __syncthreads();
    const int nkeep = nms_sweep<CN_THREADS>(sbox4, sarea, nk, CN_MASK_WPR, iou_thr, smask, skeep);
    // ordered write-out of the kept rows, one per thread (nkeep <= K < CN_THREADS)
    if (t < nkeep) {
        const int k = t, i = skeep[k];
        const unsigned long long key = dkey[i];
        const unsigned int flat = key_index(key);
        o_scores[(long long)b * out_cap + k] = key_score(key);
        o_index[(long long)b * out_cap + k] = (int)flat;
        o_cls[(long long)b * out_cap + k] = (long long)(flat / (unsigned int)(H * W));
        float* op = o_boxes + ((long long)b * out_cap + k) * 11;
#pragma unroll
        for (int q = 0; q < 11; ++q) op[q] = sbox[i][q];
    }
    if (t == 0) o_count[b] = nkeep;
}

}  // namespace vd3d

using namespace vd3d;

extern "C" long long vd3d_monoflex_decode_workspace(int B, int cap) { return (long long)B * cap * 8 + (long long)B * 4 + 64; }

extern "C" int vd3d_monoflex_decode(const float* heads, int B, int H, int W, int ncls, int cs, int hm_co, int bbox2d_co, int hps_co, int rot_co,
                                    int dim_co, int reg_co, int depth_co, int dunc_co, int cunc_co, const float* P2,
                                    float score_thr, double iou_thr, int K, float unc_lo, float unc_hi, float img_w, float img_h,
                                    int cap, void* wsp, int out_cap, float* out_scores, float* out_boxes, long long* out_cls,
                                    int* out_index, int* out_count, int* out_ncand, void* stream) {
    VD3D_REQUIRE(heads && P2 && wsp && out_scores && out_boxes && out_cls && out_index && out_count && out_ncand, "monoflex_decode: null pointer");
    VD3D_REQUIRE(B > 0 && H > 0 && W > 0 && ncls > 0 && K > 0 && K <= CN_MAXK && out_cap >= K && cap >= K && cap <= 8192, "monoflex_decode: bad shape (K <= 128, cap <= 8192)");
    VD3D_REQUIRE(score_thr > 0.f, "monoflex_decode: score_thr must be positive");
    cudaStream_t st = (cudaStream_t)stream;
    CnLayout L{cs, hm_co, bbox2d_co, hps_co, rot_co, dim_co, reg_co, depth_co, dunc_co, cunc_co};
    unsigned long long* keys = (unsigned long long*)wsp;
    int* ncand = (int*)((unsigned char*)wsp + (long long)B * cap * 8);
    VD3D_CUDA(cudaMemsetAsync(ncand, 0, sizeof(int) * B, st));
    long long total = (long long)B * ncls * H * W;
    cn_peaks_kernel<<<cdiv(total, 256), 256, 0, st>>>(heads, B, H, W, cs, hm_co, ncls, false, score_thr, cap, keys, ncand);
    VD3D_CHECK_LAUNCH("cn_peaks");
    int cp2 = next_pow2(cap);
    size_t smem = (size_t)cp2 * 8;
    VD3D_CUDA(cudaFuncSetAttribute(cn_decode_nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cn_decode_nms_kernel<<<B, CN_THREADS, smem, st>>>(heads, P2, H, W, ncls, L, cap, cp2, K, unc_lo, unc_hi, iou_thr, img_w, img_h, out_cap,
                                                     keys, ncand, out_scores, out_boxes, out_cls, out_index, out_count, out_ncand);
    VD3D_CHECK_LAUNCH("cn_decode_nms");
    return VD3D_OK;
}

extern "C" long long vd3d_km3d_decode_workspace(int B, int cap, int hp_cap) {
    return (long long)B * cap * 8 + (long long)B * 9 * hp_cap * 8 + (long long)B * 10 * 4 + 128;
}

extern "C" int vd3d_km3d_decode(const float* heads, int B, int H, int W, int ncls, int cs, int hm_co, int wh_co, int hps_co, int rot_co,
                                int dim_co, int prob_co, int reg_co, int hm_hp_co, int hp_offset_co, const float* P2,
                                float score_thr, double iou_thr, int K, float img_w, float img_h, int cap, int hp_cap, void* wsp,
                                int out_cap, float* out_scores, float* out_boxes, long long* out_cls, int* out_index, int* out_count,
                                int* out_ncand, void* stream) {
    VD3D_REQUIRE(heads && P2 && wsp && out_scores && out_boxes && out_cls && out_index && out_count && out_ncand, "km3d_decode: null pointer");
    VD3D_REQUIRE(B > 0 && H > 0 && W > 0 && ncls > 0 && K > 0 && K <= CN_MAXK && out_cap >= K && cap >= K && cap <= 8192 && hp_cap >= K && hp_cap <= 8192,
                 "km3d_decode: bad shape (K <= 128, caps <= 8192)");
    VD3D_REQUIRE(score_thr > 0.f, "km3d_decode: score_thr must be positive");
    cudaStream_t st = (cudaStream_t)stream;
    KmLayout L{cs, hm_co, wh_co, hps_co, rot_co, dim_co, prob_co, reg_co, hm_hp_co, hp_offset_co};
    unsigned char* p = (unsigned char*)wsp;
    unsigned long long* keys = (unsigned long long*)p; p += (long long)B * cap * 8;
    unsigned long long* hp_keys = (unsigned long long*)p; p += (long long)B * 9 * hp_cap * 8;
    int* ncand = (int*)p; int* hp_ncand = ncand + B;
    VD3D_CUDA(cudaMemsetAsync(ncand, 0, sizeof(int) * B * 10, st));
    // detection peaks: the reference keeps the K best then drops scores <= score_thr; pre-filtering with the threshold is equivalent, and
    // it is the only score test: every decoded peak is above score_thr
    long long total = (long long)B * ncls * H * W;
    cn_peaks_kernel<<<cdiv(total, 256), 256, 0, st>>>(heads, B, H, W, cs, hm_co, ncls, false, score_thr, cap, keys, ncand);
    VD3D_CHECK_LAUNCH("km3d_peaks");
    long long total_hp = (long long)B * 9 * H * W;
    cn_peaks_kernel<<<cdiv(total_hp, 256), 256, 0, st>>>(heads, B, H, W, cs, hm_hp_co, 9, true, 0.1f, hp_cap, hp_keys, hp_ncand);
    VD3D_CHECK_LAUNCH("km3d_hp_peaks");
    int cp2 = next_pow2(cap);
    int hp2 = next_pow2(hp_cap);
    size_t smem = (size_t)(cp2 > hp2 ? cp2 : hp2) * 8;
    VD3D_CUDA(cudaFuncSetAttribute(km3d_decode_nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    km3d_decode_nms_kernel<<<B, CN_THREADS, smem, st>>>(heads, P2, H, W, ncls, L, cap, cp2, hp_cap, hp2, K, iou_thr, img_w, img_h,
                                                       out_cap, keys, ncand, hp_keys, hp_ncand, out_scores, out_boxes, out_cls, out_index,
                                                       out_count, out_ncand);
    VD3D_CHECK_LAUNCH("km3d_decode_nms");
    return VD3D_OK;
}
