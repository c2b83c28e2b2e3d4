// Anchor filtering, box decode, clipping and NMS for the anchor-based 3-D head, batched, fixed capacity, no host
// round trips (the reference does ~30 tiny eager kernels and >= 6 D2H syncs per image,
// R/heads/detection_3d_head.py:341-400).
//
// Bit-exactness: index sets (useful mask, score threshold, prior validity, NMS keep) are decided by fp32
// comparisons whose operands are computed with the SAME operation order as the reference's eager ops and with
// FMA contraction disabled (explicit __fmul_rn/__fadd_rn/__fdiv_rn), so they only differ where the CUDA libm
// (expf/atan2f) differs from the host libm by an ulp on a knife edge.
#include "decode_common.cuh"
#include <cstring>

namespace vd3d {

// ---------------------------------------------------------------------------------------------------------
// useful mask (R/heads/anchors.py:93-111)
//   x3d = (xc*z - cx*z)/fy ; y3d = (yc*z - cy*z)/fy ; mask = any_t( y3d > ymin && y3d < ymax && |x3d| < xthr )
//   xc = mean(x1, x2) computed by torch as (x1 + x2) / 2
// ---------------------------------------------------------------------------------------------------------
__global__ void anchor_mask_kernel(const float* __restrict__ anchors, const float* __restrict__ means_z, const float* __restrict__ P2,
                                   int B, int N, int T, float y_min, float y_max, float x_thr, uint8_t* __restrict__ mask) {
    long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)B * N) return;
    int n = (int)(idx % N), b = (int)(idx / N);
    float4 a = ldg4(anchors + 4 * (long long)n);
    float xc = __fdiv_rn(add(a.x, a.z), 2.0f);
    float yc = __fdiv_rn(add(a.y, a.w), 2.0f);
    const float* P = P2 + 12 * b;
    float fy = P[5], cy = P[6], cx = P[2];
    bool any = false;
    for (int t = 0; t < T; ++t) {
        float z = __ldg(means_z + (long long)t * N + n);
        float x3 = __fdiv_rn(sub(mul(xc, z), mul(cx, z)), fy);
        float y3 = __fdiv_rn(sub(mul(yc, z), mul(cy, z)), fy);
        any = any || ((y3 > y_min) && (y3 < y_max) && (fabsf(x3) < x_thr));
    }
    mask[idx] = any ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------------------
// stage 1: score + threshold + validity -> unordered candidate list (atomic compaction).  The order is fixed
// afterwards by the sort key (score desc, anchor index asc) == torchvision's stable descending sort of the
// index-ordered candidate list.
// workspace layout per image: keys u64[cap], boxes f32[cap][11], labels i32[cap]
// ---------------------------------------------------------------------------------------------------------
struct DecodeWs {
    unsigned long long* keys;   // [B][cap]
    float* boxes;               // [B][cap][11]
    int* labels;                // [B][cap]
    int* ncand;                 // [B]
};

// The candidate test of the decoder: the first maximum over the classes of sigmoid(cls) (torch.max over dim) and whether it clears the
// score threshold.  decode_candidates_kernel and reg_candidates_kernel both call it, so the regression rows computed for the decoder are
// always a superset of the rows it reads.
__device__ __forceinline__ bool anchor_score(const float* cp, int ncls, float score_thr, float& best, int& label) {
    best = -1.f; label = 0;
    for (int c = 0; c < ncls; ++c) {
        float p = sigmoid_ref(__ldg(cp + c));
        if (p > best) { best = p; label = c; }     // first maximum wins (torch.max over dim)
    }
    return best > score_thr;
}

// The (pixel, anchor group) pairs whose regression values the decoder may read: some anchor of the group is inside the anchor mask and
// passes anchor_score.  The decoder's z_mean > 0 test is not applied: the list is a superset of what it reads, never a subset.
// One thread per (image, pixel, group); pair -> list[group][slot] = b * P + pixel, counts[group] (zeroed by the caller) = slots used.
// The capacity of each group is B * P, so the list cannot overflow.  The order of the slots is not fixed: the gathered conv computes
// every row on its own.
// pixmap (optional, zeroed by the caller): byte b * P + pixel set when the pixel is listed in some group.
__global__ void reg_candidates_kernel(const float* __restrict__ cls, const uint8_t* __restrict__ mask, int B, int P, int A, int ncls,
                                      float score_thr, int ga, int groups, int32_t* __restrict__ list, int32_t* __restrict__ counts,
                                      uint8_t* __restrict__ pixmap) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)B * P * groups) return;
    const int grp = (int)(idx % groups);
    const long long pix = idx / groups;                       // b * P + pixel
    bool any = false;
    for (int a = grp * ga; a < min(A, (grp + 1) * ga) && !any; ++a) {
        const long long n = pix * A + a;                      // b * N + anchor
        float best; int label;
        any = mask[n] && anchor_score(cls + n * (ncls + 1), ncls, score_thr, best, label);
    }
    if (!any) return;
    const int slot = atomicAdd(counts + grp, 1);
    list[(long long)grp * B * P + slot] = (int32_t)pix;
    if (pixmap) pixmap[pix] = 1;
}

// Tile lists of the regression tower (vd3d_reg_tower_tiles).  Block d - 1 builds depth d: S_d = the pixels within d 3x3 steps of a candidate
// pixel (a (2 d + 1)^2 window, clipped to the image: separable, rows then columns, in shared memory), and per image the 8 x 16 tiles whose
// rows start at the first row of S_d and which hold a pixel of S_d, listed in the order image, tile row, tile column (warp 0 compacts the
// tile flags 32 at a time), so the list does not depend on the schedule.
__global__ void reg_tower_tiles_kernel(const uint8_t* __restrict__ cand, int B, int H, int W, uint8_t* __restrict__ smaps,
                                       int4* __restrict__ tiles, int cap, int32_t* __restrict__ counts) {
    extern __shared__ uint8_t sh[];
    const int d = (int)blockIdx.x + 1, HW = H * W, TW = (W + 15) / 16, TH = (H + 7) / 8 + 1;
    uint8_t* rows = sh;                                       // [H][W] candidates dilated along the row
    uint8_t* set = sh + HW;                                   // [H][W] S_d
    int* flag = reinterpret_cast<int*>(sh + ((2 * HW + 15) & ~15));     // [TH][TW]
    __shared__ int ymin;
    int base = 0;                                             // (warp 0) entries listed so far
    uint8_t* smap = smaps + (long long)blockIdx.x * B * HW;
    int4* list = tiles + (long long)blockIdx.x * cap;
    for (int b = 0; b < B; ++b) {
        const uint8_t* c = cand + (long long)b * HW;
        if (threadIdx.x == 0) ymin = H;
        for (int i = threadIdx.x; i < TH * TW; i += blockDim.x) flag[i] = 0;
        for (int i = threadIdx.x; i < HW; i += blockDim.x) {
            const int y = i / W, x = i - y * W;
            uint8_t v = 0;
            for (int xx = max(0, x - d); xx <= min(W - 1, x + d); ++xx) v |= c[y * W + xx];
            rows[i] = v;
        }
        __syncthreads();
        for (int i = threadIdx.x; i < HW; i += blockDim.x) {
            const int y = i / W, x = i - y * W;
            uint8_t v = 0;
            for (int yy = max(0, y - d); yy <= min(H - 1, y + d); ++yy) v |= rows[yy * W + x];
            v = v ? 1 : 0;
            set[i] = v;
            smap[(long long)b * HW + i] = v;
            if (v) atomicMin(&ymin, y);
        }
        __syncthreads();
        const int y0 = ymin;
        for (int i = threadIdx.x; i < HW; i += blockDim.x) {
            const int y = i / W, x = i - y * W;
            if (set[i]) flag[((y - y0) >> 3) * TW + (x >> 4)] = 1;
        }
        __syncthreads();
        if (threadIdx.x < 32) {
            for (int t0 = 0; t0 < TH * TW; t0 += 32) {
                const int t = t0 + (int)threadIdx.x;
                const bool on = t < TH * TW && flag[t];
                const unsigned bal = __ballot_sync(0xffffffffu, on);
                if (on) {
                    const int ty = t / TW, tx = t - ty * TW;
                    list[base + __popc(bal & ((1u << threadIdx.x) - 1u))] = make_int4(b, y0 + 8 * ty, 16 * tx, 0);
                }
                base += __popc(bal);
            }
        }
        __syncthreads();                                      // rows / set / flag / ymin are reused by the next image
    }
    if (threadIdx.x == 0) counts[blockIdx.x] = base;
}

__global__ void decode_candidates_kernel(const float* __restrict__ cls, const float* __restrict__ reg, const float* __restrict__ anchors,
                                         const float* __restrict__ mean_std, const uint8_t* __restrict__ mask,
                                         int B, int N, int ncls, int T, float score_thr, float img_w, float img_h, int cap, DecodeWs ws) {
    long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)B * N) return;
    int n = (int)(idx % N), b = (int)(idx / N);
    if (!mask[idx]) return;
    const float* cp = cls + idx * (ncls + 1);
    float best; int label;
    if (!anchor_score(cp, ncls, score_thr, best, label)) return;
    const float* ms = mean_std + ((long long)n * T + label) * 12;   // [6][2]
    float z_mean = __ldg(ms + 0);
    if (!(z_mean > 0.f)) return;                                    // `mask = selected_mean_std[:,0,0] > 0` (:242)
    float alpha_score = sigmoid_ref(__ldg(cp + ncls));

    float4 a = ldg4(anchors + 4 * (long long)n);
    const float* d = reg + idx * 12;
    float widths = sub(a.z, a.x), heights = sub(a.w, a.y);
    float ctr_x = add(a.x, mul(0.5f, widths)), ctr_y = add(a.y, mul(0.5f, heights));
    float dx = mul(__ldg(d + 0), 0.1f), dy = mul(__ldg(d + 1), 0.1f);
    float dw = mul(__ldg(d + 2), 0.2f), dh = mul(__ldg(d + 3), 0.2f);
    float pcx = add(ctr_x, mul(dx, widths)), pcy = add(ctr_y, mul(dy, heights));
    float pw = mul(expf(dw), widths), ph = mul(expf(dh), heights);
    float x1 = sub(pcx, mul(0.5f, pw)), y1 = sub(pcy, mul(0.5f, ph));
    float x2 = add(pcx, mul(0.5f, pw)), y2 = add(pcy, mul(0.5f, ph));
    float cx1 = add(ctr_x, mul(mul(__ldg(d + 4), 0.1f), widths));
    float cy1 = add(ctr_y, mul(mul(__ldg(d + 5), 0.1f), heights));
    float z = add(mul(__ldg(d + 6), __ldg(ms + 1)), z_mean);
    float sn = add(mul(__ldg(d + 7), __ldg(ms + 3)), __ldg(ms + 2));
    float cs = add(mul(__ldg(d + 8), __ldg(ms + 5)), __ldg(ms + 4));
    float alpha = __fdiv_rn(atan2f(sn, cs), 2.0f);
    float w3 = add(mul(__ldg(d + 9), __ldg(ms + 7)), __ldg(ms + 6));
    float h3 = add(mul(__ldg(d + 10), __ldg(ms + 9)), __ldg(ms + 8));
    float l3 = add(mul(__ldg(d + 11), __ldg(ms + 11)), __ldg(ms + 10));
    if (alpha_score < 0.5f) alpha = add(alpha, 3.14159265358979323846f);   // `+= np.pi` on an f32 tensor
    // ClipBoxes (R/utils/utils.py:181-196)
    x1 = fmaxf(x1, 0.f); y1 = fmaxf(y1, 0.f); x2 = fminf(x2, img_w); y2 = fminf(y2, img_h);

    int slot = atomicAdd(ws.ncand + b, 1);
    if (slot >= cap) return;                       // overflow: flagged through ncand > cap
    ws.keys[(long long)b * cap + slot] = score_key(best, (unsigned int)n);     // best > score_thr > 0
    float* bp = ws.boxes + ((long long)b * cap + slot) * 11;
    bp[0] = x1; bp[1] = y1; bp[2] = x2; bp[3] = y2; bp[4] = cx1; bp[5] = cy1; bp[6] = z; bp[7] = w3; bp[8] = h3; bp[9] = l3; bp[10] = alpha;
    ws.labels[(long long)b * cap + slot] = label;
}

// ---------------------------------------------------------------------------------------------------------
// stage 2 (one CTA per image): bitonic sort of (key, slot) in shared memory, greedy NMS (nms_sweep), ordered write-out.
// ---------------------------------------------------------------------------------------------------------
constexpr int NMS_THREADS = 1024;

__global__ void __launch_bounds__(NMS_THREADS) sort_nms_kernel(DecodeWs ws, int cap, int cap_pow2, double iou_thr,
                                                                float* __restrict__ out_scores, float* __restrict__ out_boxes,
                                                                int64_t* __restrict__ out_cls, int32_t* __restrict__ out_anchor,
                                                                int32_t* __restrict__ out_count, int32_t* __restrict__ out_ncand) {
    extern __shared__ __align__(16) unsigned char sm_raw[];
    unsigned long long* skey = reinterpret_cast<unsigned long long*>(sm_raw);            // [cap_pow2]
    unsigned long long* smask = skey + cap_pow2;                                         // [64][cap_pow2 / 64]: suppression bits of one 64-row block
    float4* sbox = reinterpret_cast<float4*>(smask + cap_pow2);                          // [cap_pow2]
    int* sslot = reinterpret_cast<int*>(sbox + cap_pow2);                                // [cap_pow2]
    float* sarea = reinterpret_cast<float*>(sslot + cap_pow2);                           // [cap_pow2]
    int* skeep = reinterpret_cast<int*>(sarea + cap_pow2);                               // [cap_pow2] sorted positions of the kept boxes
    const int b = blockIdx.x, t = threadIdx.x;
    const int n = ws.ncand[b];
    if (t == 0) out_ncand[b] = n;
    if (n > cap) { if (t == 0) out_count[b] = -1; return; }
    const int np2 = next_pow2(n, 64);               // sort size (the padding keys ~0 sort to the end)

    for (int i = t; i < np2; i += NMS_THREADS) {
        skey[i] = (i < n) ? ws.keys[(long long)b * cap + i] : ~0ull;
        sslot[i] = i;
    }
    __syncthreads();
    block_sort<NMS_THREADS, true>(skey, sslot, np2);
    for (int i = t; i < n; i += NMS_THREADS) {
        const float* bp = ws.boxes + ((long long)b * cap + sslot[i]) * 11;
        float4 bx = make_float4(bp[0], bp[1], bp[2], bp[3]);
        sbox[i] = bx;
        sarea[i] = box_area(bx);
    }
    __syncthreads();
    const int nkeep = nms_sweep<NMS_THREADS>(sbox, sarea, n, cap_pow2 >> 6, iou_thr, smask, skeep);
    // ordered write-out of the kept boxes, all threads
    for (int k = t; k < nkeep; k += NMS_THREADS) {
        const int i = skeep[k];
        const int slot = sslot[i];
        const unsigned long long key = skey[i];
        out_scores[(long long)b * cap + k] = key_score(key);
        out_anchor[(long long)b * cap + k] = (int)key_index(key);
        out_cls[(long long)b * cap + k] = (int64_t)ws.labels[(long long)b * cap + slot];
        const float* bp = ws.boxes + ((long long)b * cap + slot) * 11;
        float* op = out_boxes + ((long long)b * cap + k) * 11;
#pragma unroll
        for (int q = 0; q < 11; ++q) op[q] = bp[q];
    }
    if (t == 0) out_count[b] = nkeep;
}

// ---------------------------------------------------------------------------------------------------------
// RetinaNet 2-D decode (RetinanetHead.get_bboxes, R/heads/retinanet_head.py:257-307), batched, no host sync:
//   (1) retina_score_kernel: per anchor, max over classes of sigmoid(cls) (first maximum wins) -> 32-bit key ~bits(score) (ascending =
//       better) and the label;
//   (2) retina_select_kernel (one CTA per image): the k = min(nms_pre, N) smallest keys by an 8-bit radix select (4 histogram passes),
//       ties at the k-th key resolved by anchor index (ascending, an ordered block scan), then the _decode of the selected rows (:227-255,
//       no ClipBoxes) into the sort_nms_kernel workspace with box columns 4..10 zero;
//   (3) sort_nms_kernel: sort by (score desc, index asc) + greedy class-agnostic NMS;
//   (4) retina_thresh_kernel: the post-NMS score threshold, a prefix of the score-ordered kept rows, as a count.
// Head outputs are per pyramid level (NHWC [B][pix_l][cs]): anchor n of level l at local index j = n - off_l is pixel j / A, channel
// (j % A) * C + c.
// ---------------------------------------------------------------------------------------------------------
constexpr int RETINA_MAX_LEVELS = 8;
struct RetinaLevels {
    const float* cls[RETINA_MAX_LEVELS];
    const float* reg[RETINA_MAX_LEVELS];
    int pix[RETINA_MAX_LEVELS];
    int off[RETINA_MAX_LEVELS + 1];          // first anchor of level l (off[L] = N)
    int L, A, cls_cs, reg_cs;
};

__device__ __forceinline__ long long retina_elem(const RetinaLevels& lv, int b, int n, int cs, int per, int& l_out) {
    int l = 0;
    while (l + 1 < lv.L && n >= lv.off[l + 1]) ++l;
    const int j = n - lv.off[l];
    const int px = j / lv.A, a = j - px * lv.A;
    l_out = l;
    return ((long long)b * lv.pix[l] + px) * cs + (long long)a * per;
}

__global__ void retina_score_kernel(RetinaLevels lv, int B, int N, int ncls, unsigned int* __restrict__ keys, uint8_t* __restrict__ labels) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)B * N) return;
    const int n = (int)(idx % N), b = (int)(idx / N);
    int l;
    const long long e = retina_elem(lv, b, n, lv.cls_cs, ncls, l);
    const float* cp = lv.cls[l] + e;
    float best = -1.f; int label = 0;
    for (int c = 0; c < ncls; ++c) {
        const float p = sigmoid_ref(__ldg(cp + c));
        if (p > best) { best = p; label = c; }
    }
    keys[idx] = (unsigned int)(score_key(best, 0u) >> 32);     // the score half of the sort key (sigmoid >= +0)
    labels[idx] = (uint8_t)label;
}

constexpr int SEL_THREADS = 1024;

// exclusive prefix of `flag` over the block (thread order) and the block total
__device__ __forceinline__ int block_excl_scan(bool flag, int* s_warp, int& total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned int bal = __ballot_sync(0xffffffffu, flag);
    const int in_warp = __popc(bal & ((1u << lane) - 1u));
    if (lane == 0) s_warp[warp] = __popc(bal);
    __syncthreads();
    if (warp == 0) {
        const int v = s_warp[lane];
        int x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
        s_warp[32 + lane] = x - v;
        if (lane == 31) s_warp[64] = x;
    }
    __syncthreads();
    const int r = s_warp[32 + warp] + in_warp;
    total = s_warp[64];
    __syncthreads();
    return r;
}

__global__ void __launch_bounds__(SEL_THREADS) retina_select_kernel(RetinaLevels lv, const unsigned int* __restrict__ keys, const uint8_t* __restrict__ labels,
                                                                    const float* __restrict__ anchors, int N, int k, float4 mean, float4 std, int cap, DecodeWs ws) {
    __shared__ int hist[256];
    __shared__ int s_warp[65];
    __shared__ unsigned int s_prefix;
    __shared__ int s_need;
    const int b = blockIdx.x, t = threadIdx.x;
    const unsigned int* kp = keys + (long long)b * N;
    // ---- radix select: T = the k-th smallest key, `need` = how many keys equal to T are taken ----
    unsigned int T = 0xffffffffu;
    int need = 0;
    if (k < N) {
        if (t == 0) { s_prefix = 0; s_need = k; }
        __syncthreads();
        for (int shift = 24; shift >= 0; shift -= 8) {
            for (int i = t; i < 256; i += SEL_THREADS) hist[i] = 0;
            __syncthreads();
            const unsigned int prefix = s_prefix;
            const unsigned int hmask = shift == 24 ? 0u : (0xffffffffu << (shift + 8));
            for (int i = t; i < N; i += SEL_THREADS) {
                const unsigned int key = __ldg(kp + i);
                if ((key & hmask) == prefix) atomicAdd(&hist[(key >> shift) & 255], 1);
            }
            __syncthreads();
            if (t == 0) {
                int rem = s_need, d = 0;
                while (hist[d] < rem) { rem -= hist[d]; ++d; }
                s_prefix = prefix | ((unsigned int)d << shift);
                s_need = rem;
            }
            __syncthreads();
        }
        T = s_prefix;
        need = s_need;
    }
    // ---- ordered compaction: every key < T, and the first `need` keys == T in anchor order; decode into the NMS workspace ----
    int taken_ties = 0, slot0 = 0;
    for (int base = 0; base < N; base += SEL_THREADS) {
        const int n = base + t;
        const unsigned int key = n < N ? __ldg(kp + n) : 0xffffffffu;
        const bool tie = n < N && k < N && key == T;
        int ntie;
        const int tie_rank = block_excl_scan(tie, s_warp, ntie);
        const bool sel = n < N && (k >= N || key < T || (tie && taken_ties + tie_rank < need));
        int nsel;
        const int pos = slot0 + block_excl_scan(sel, s_warp, nsel);
        taken_ties += ntie;
        slot0 += nsel;
        if (!sel || pos >= cap) continue;
        int l;
        const float* rp = lv.reg[0];
        {
            const long long e = retina_elem(lv, b, n, lv.reg_cs, 4, l);
            rp = lv.reg[l] + e;
        }
        const float4 a = ldg4(anchors + 4 * (long long)n);
        const float dx = add(mul(__ldg(rp + 0), std.x), mean.x), dy = add(mul(__ldg(rp + 1), std.y), mean.y);
        const float dw = add(mul(__ldg(rp + 2), std.z), mean.z), dh = add(mul(__ldg(rp + 3), std.w), mean.w);
        const float px = mul(add(a.x, a.z), 0.5f), py = mul(add(a.y, a.w), 0.5f);
        const float pw = sub(a.z, a.x), ph = sub(a.w, a.y);
        const float gw = mul(pw, expf(dw)), gh = mul(ph, expf(dh));
        const float gx = add(px, mul(pw, dx)), gy = add(py, mul(ph, dy));
        const long long o = (long long)b * cap + pos;
        ws.keys[o] = score_key(key_score((unsigned long long)key << 32), (unsigned int)n);
        float* bp = ws.boxes + o * 11;
        bp[0] = sub(gx, mul(gw, 0.5f)); bp[1] = sub(gy, mul(gh, 0.5f)); bp[2] = add(gx, mul(gw, 0.5f)); bp[3] = add(gy, mul(gh, 0.5f));
#pragma unroll
        for (int q = 4; q < 11; ++q) bp[q] = 0.f;
        ws.labels[o] = (int)labels[(long long)b * N + n];
    }
    if (t == 0) ws.ncand[b] = slot0;
}

// post-NMS `max_score > score_thr` (retinanet_head.py:295-304): the kept rows are in descending score order, so the survivors are a prefix
__global__ void retina_thresh_kernel(const float* __restrict__ scores, int cap, float score_thr, int32_t* __restrict__ count) {
    __shared__ int s_n;
    const int b = blockIdx.x;
    const int n = count[b];
    if (n < 0) return;
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    int c = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) c += scores[(long long)b * cap + i] > score_thr;
    atomicAdd(&s_n, c);
    __syncthreads();
    if (threadIdx.x == 0) count[b] = s_n;
}

// fixed-capacity detection record block for the multi-GPU all-gather: rec[b] = [count | kmax x (11 box floats, score, class)]
__global__ void pack_records_kernel(const float* __restrict__ scores, const float* __restrict__ boxes, const int64_t* __restrict__ cls,
                                    const int32_t* __restrict__ count, int cap, int kmax, float* __restrict__ rec, const int* __restrict__ range_flag) {
    const int b = blockIdx.x;
    int n = count[b];
    if (range_flag && *range_flag) n = -2;                            // -2: an activation left the fp16 range of the tensor-core engine (results invalid)
    float* r = rec + (long long)b * (1 + kmax * 13);
    if (threadIdx.x == 0) r[0] = (n > kmax) ? -1.0f : (float)n;       // -1: capacity overflow (also n == -1 from the decode stage)
    const int m = n < 0 ? 0 : (n > kmax ? 0 : n);
    for (int i = threadIdx.x; i < kmax * 13; i += blockDim.x) {
        int k = i / 13, q = i - k * 13;
        float v = 0.f;
        if (k < m) v = (q < 11) ? boxes[((long long)b * cap + k) * 11 + q] : (q == 11 ? scores[(long long)b * cap + k] : (float)cls[(long long)b * cap + k]);
        r[1 + i] = v;
    }
}

}  // namespace vd3d

using namespace vd3d;

extern "C" int vd3d_pack_records(const float* scores, const float* boxes, const int64_t* cls, const int32_t* count, int B, int cap, int kmax,
                                 float* rec, void* stream) {
    VD3D_REQUIRE(scores && boxes && cls && count && rec && B > 0 && cap > 0 && kmax > 0, "pack_records: bad args");
    pack_records_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(scores, boxes, cls, count, cap, kmax, rec, fp16_range_flag());
    VD3D_CHECK_LAUNCH("pack_records");
    return VD3D_OK;
}

extern "C" int vd3d_anchor_mask(const float* anchors, const float* means_z, const float* P2, int B, int N, int T,
                                float y_min, float y_max, float x_thr, uint8_t* mask, void* stream) {
    VD3D_REQUIRE(anchors && means_z && P2 && mask && B > 0 && N > 0 && T > 0, "anchor_mask: bad args");
    anchor_mask_kernel<<<cdiv((long long)B * N, 256), 256, 0, (cudaStream_t)stream>>>(anchors, means_z, P2, B, N, T, y_min, y_max, x_thr, mask);
    VD3D_CHECK_LAUNCH("anchor_mask");
    return VD3D_OK;
}

extern "C" int vd3d_reg_candidates(const float* cls, const uint8_t* mask, int B, int P, int A, int ncls, float score_thr, int group_anchors,
                                   int32_t* list, int32_t* counts, uint8_t* pixmap, void* stream) {
    VD3D_REQUIRE(cls && mask && list && counts && B > 0 && P > 0 && A > 0 && ncls > 0 && group_anchors > 0, "reg_candidates: bad args");
    VD3D_REQUIRE((long long)B * P * A < (1LL << 31), "reg_candidates: too many anchors for the 32-bit list");
    const int groups = cdiv(A, group_anchors);
    cudaStream_t st = (cudaStream_t)stream;
    VD3D_CUDA(cudaMemsetAsync(counts, 0, sizeof(int32_t) * groups, st));
    if (pixmap) VD3D_CUDA(cudaMemsetAsync(pixmap, 0, (size_t)B * P, st));
    reg_candidates_kernel<<<cdiv((long long)B * P * groups, 256), 256, 0, st>>>(cls, mask, B, P, A, ncls, score_thr, group_anchors, groups, list, counts,
                                                                               pixmap);
    VD3D_CHECK_LAUNCH("reg_candidates");
    return VD3D_OK;
}

extern "C" int vd3d_reg_tower_tile_cap(int B, int H, int W) { return B * (cdiv(H, 8) + 1) * cdiv(W, 16); }

// shared memory of reg_tower_tiles_kernel: two [H][W] byte maps and the [cdiv(H, 8) + 1][cdiv(W, 16)] tile flags
static size_t tower_tiles_smem(int H, int W) { return (size_t)((2 * H * W + 15) & ~15) + sizeof(int) * (cdiv(H, 8) + 1) * cdiv(W, 16); }

extern "C" int vd3d_reg_tower_tiles(const uint8_t* cand, int B, int H, int W, int D, uint8_t* smaps, int32_t* tiles, int32_t* counts, void* stream) {
    VD3D_REQUIRE(cand && smaps && tiles && counts && B > 0 && H > 0 && W > 0 && D >= 1 && D <= 16, "reg_tower_tiles: bad args");
    VD3D_REQUIRE(((uintptr_t)tiles & 15) == 0, "reg_tower_tiles: the tile list must be 16-byte aligned");
    VD3D_REQUIRE(tower_tiles_smem(H, W) <= 48 * 1024, "reg_tower_tiles: a %dx%d map does not fit the kernel's shared memory", H, W);
    reg_tower_tiles_kernel<<<D, 512, tower_tiles_smem(H, W), (cudaStream_t)stream>>>(cand, B, H, W, smaps, reinterpret_cast<int4*>(tiles),
                                                                                   vd3d_reg_tower_tile_cap(B, H, W), counts);
    VD3D_CHECK_LAUNCH("reg_tower_tiles");
    return VD3D_OK;
}

extern "C" long long vd3d_decode_nms_workspace(int B, int cap) {
    // keys u64 + boxes 11 f32 + labels i32 per slot, + ncand i32 per image (16-byte aligned blocks)
    long long per = (long long)cap * (8 + 44 + 4);
    return (long long)B * per + 16 * ((B * 4 + 15) / 16) + 64;
}

static DecodeWs decode_ws(void* wsp, int B, int cap) {
    DecodeWs ws;
    unsigned char* p = (unsigned char*)wsp;
    ws.keys = (unsigned long long*)p; p += (long long)B * cap * 8;
    ws.boxes = (float*)p; p += (long long)B * cap * 44;
    ws.labels = (int*)p; p += (long long)B * cap * 4;
    ws.ncand = (int*)p;
    return ws;
}

static int launch_sort_nms(const DecodeWs& ws, int B, int cap, double iou_thr, float* out_scores, float* out_boxes, int64_t* out_cls,
                           int32_t* out_anchor, int32_t* out_count, int32_t* out_ncand, cudaStream_t st) {
    const int cp2 = next_pow2(cap, 64);          // the 64-row bit-matrix blocks of the NMS sweep
    const size_t smem = (size_t)cp2 * (8 + 8 + 16 + 4 + 4 + 4) + 16;
    VD3D_CUDA(cudaFuncSetAttribute(sort_nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    sort_nms_kernel<<<B, NMS_THREADS, smem, st>>>(ws, cap, cp2, iou_thr, out_scores, out_boxes, out_cls, out_anchor, out_count, out_ncand);
    VD3D_CHECK_LAUNCH("sort_nms");
    return VD3D_OK;
}

extern "C" int vd3d_decode_nms(const float* cls, const float* reg, const float* anchors, const float* mean_std,
                               const uint8_t* mask, int B, int N, int ncls, int T, float score_thr, double iou_thr,
                               float img_w, float img_h, int cap, void* wsp,
                               float* out_scores, float* out_boxes, int64_t* out_cls, int32_t* out_anchor,
                               int32_t* out_count, int32_t* out_ncand, void* stream) {
    VD3D_REQUIRE(cls && reg && anchors && mean_std && mask && wsp && out_scores && out_boxes && out_cls && out_anchor && out_count && out_ncand,
                 "decode_nms: null pointer");
    VD3D_REQUIRE(B > 0 && N > 0 && ncls > 0 && ncls <= T && cap > 0 && cap <= 4096, "decode_nms: bad shape (cap must be <= 4096)");
    VD3D_REQUIRE(score_thr > 0.f, "decode_nms: score_thr must be positive (sort key relies on positive scores)");
    cudaStream_t st = (cudaStream_t)stream;
    const DecodeWs ws = decode_ws(wsp, B, cap);
    VD3D_CUDA(cudaMemsetAsync(ws.ncand, 0, sizeof(int) * B, st));
    decode_candidates_kernel<<<cdiv((long long)B * N, 256), 256, 0, st>>>(cls, reg, anchors, mean_std, mask, B, N, ncls, T,
                                                                         score_thr, img_w, img_h, cap, ws);
    VD3D_CHECK_LAUNCH("decode_candidates");
    return launch_sort_nms(ws, B, cap, iou_thr, out_scores, out_boxes, out_cls, out_anchor, out_count, out_ncand, st);
}

extern "C" long long vd3d_retina_decode_workspace(int B, int N, int cap) {
    // the vd3d_decode_nms workspace, then keys u32 [B][N] and labels u8 [B][N]
    const long long nms = vd3d_decode_nms_workspace(B, cap);
    return nms + ((long long)B * N * 4 + 15) / 16 * 16 + (long long)B * N + 64;
}

extern "C" int vd3d_retina_decode(int L, const void* const* cls_levels, const void* const* reg_levels, const int* level_pix, int cls_cs, int reg_cs,
                                  const float* anchors, int B, int N, int A, int ncls, int nms_pre, const float* means4, const float* stds4,
                                  float score_thr, double iou_thr, int cap, void* wsp,
                                  float* out_scores, float* out_boxes, int64_t* out_cls, int32_t* out_anchor,
                                  int32_t* out_count, int32_t* out_ncand, void* stream) {
    VD3D_REQUIRE(cls_levels && reg_levels && level_pix && anchors && means4 && stds4 && wsp && out_scores && out_boxes && out_cls && out_anchor &&
                 out_count && out_ncand, "retina_decode: null pointer");
    VD3D_REQUIRE(L >= 1 && L <= RETINA_MAX_LEVELS && B > 0 && N > 0 && A > 0 && ncls > 0 && ncls <= 255 && cls_cs >= A * ncls && reg_cs >= A * 4,
                 "retina_decode: bad shape (L=%d A=%d ncls=%d cls_cs=%d reg_cs=%d)", L, A, ncls, cls_cs, reg_cs);
    const int k = (nms_pre > 0 && N > nms_pre) ? nms_pre : N;
    VD3D_REQUIRE(cap > 0 && cap <= 4096 && k <= cap, "retina_decode: %d candidates exceed the NMS capacity %d (<= 4096)", k, cap);
    RetinaLevels lv;
    memset(&lv, 0, sizeof(lv));
    lv.L = L; lv.A = A; lv.cls_cs = cls_cs; lv.reg_cs = reg_cs;
    lv.off[0] = 0;
    for (int l = 0; l < L; ++l) {
        VD3D_REQUIRE(cls_levels[l] && reg_levels[l] && level_pix[l] > 0, "retina_decode: level %d is empty", l);
        lv.cls[l] = (const float*)cls_levels[l]; lv.reg[l] = (const float*)reg_levels[l]; lv.pix[l] = level_pix[l];
        lv.off[l + 1] = lv.off[l] + level_pix[l] * A;
    }
    VD3D_REQUIRE(lv.off[L] == N, "retina_decode: the levels hold %d anchors, N = %d", lv.off[L], N);
    cudaStream_t st = (cudaStream_t)stream;
    const DecodeWs ws = decode_ws(wsp, B, cap);
    unsigned char* q = (unsigned char*)wsp + vd3d_decode_nms_workspace(B, cap);
    unsigned int* keys = (unsigned int*)q;
    uint8_t* labels = q + ((long long)B * N * 4 + 15) / 16 * 16;
    retina_score_kernel<<<cdiv((long long)B * N, 256), 256, 0, st>>>(lv, B, N, ncls, keys, labels);
    VD3D_CHECK_LAUNCH("retina_score");
    retina_select_kernel<<<B, SEL_THREADS, 0, st>>>(lv, keys, labels, anchors, N, k, make_float4(means4[0], means4[1], means4[2], means4[3]),
                                                    make_float4(stds4[0], stds4[1], stds4[2], stds4[3]), cap, ws);
    VD3D_CHECK_LAUNCH("retina_select");
    const int e = launch_sort_nms(ws, B, cap, iou_thr, out_scores, out_boxes, out_cls, out_anchor, out_count, out_ncand, st);
    if (e != VD3D_OK) return e;
    retina_thresh_kernel<<<B, 256, 0, st>>>(out_scores, cap, score_thr, out_count);
    VD3D_CHECK_LAUNCH("retina_thresh");
    return VD3D_OK;
}
