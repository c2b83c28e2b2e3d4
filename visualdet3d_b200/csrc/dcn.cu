// Deformable convolution v1 / v2 (R/lib/ops/dcn): deformable (modulated) im2col on NHWC activations.
//
//   col[b,ho,wo, k*C + c] = mask[b,ho,wo,k] * bilinear(x[b,:,:,c], ho*s - pad + kh*dil + dh_k, wo*s - pad + kw*dil + dw_k)
//
// with the reference's sampling rule (deform_conv_cuda_kernel.cu:467-497,570-633): a tap contributes only if
// h > -1 && w > -1 && h < H && w < W; the four neighbours are individually zero outside the image.  The K order
// (tap-major, channel-minor) is the conv engines' weight order, so the GEMM that follows is a plain 1x1 convolution on the
// wgmma engine (the `lo` companion of the columns is produced here for free).  Sampling coordinates and weights are
// computed once per (pixel, tap) and shared by all channels: one CTA = 32 pixels x all taps, threads sweep channel quads.
// HBM-bound gather: reads x once (L2 serves the 9x tap reuse), writes KH*KW*C floats (+lo) per pixel.
#include "common.cuh"
#include <cuda_fp16.h>

namespace vd3d {

struct DcnParams {
    const float* x; int B, H, W, C, x_cs, x_co;
    const float* off; int off_cs, off_co;           // NHWC [B][Ho][Wo][..]: channel off_co + g*2*K + 2*k (+1) = (dh, dw) of tap k, group g
    const float* msk; int msk_cs, msk_co;           // NHWC: channel msk_co + g*K + k ; nullptr -> DCNv1 (mask == 1)
    int mask_sigmoid;                               // apply sigmoid to the mask channel (fuses torch.sigmoid, deform_conv.py:463)
    int KH, KW, stride, pad, dil, dg;
    int Ho, Wo;
    float* col; float* col_lo; int col_cs;          // [B*Ho*Wo][col_cs], channels [0, KH*KW*C)
    __half* col_h16_hi; __half* col_h16_lo;         // optional fp16 (hi, lo) planes of the columns (same pitch): what the fp16-split GEMM reads
    int* range_flag;                                // fp16-range guard (common.cuh)
    int k_order;                                    // column order: 0 = tap * C + c (the reference's `columns` transposed), 1 = (chunk64 * K + tap) * 64 + c % 64
};

constexpr int DCN_PIX = 32;       // pixels per CTA
constexpr int DCN_THREADS = 256;
constexpr int DCN_MAXK = 49;      // up to 7x7 taps

__global__ void __launch_bounds__(DCN_THREADS) deform_im2col_kernel(const DcnParams p) {
    __shared__ int s_base[DCN_PIX][DCN_MAXK][2];     // (h_low * W + w_low), validity bits of the 4 neighbours (bit 4 = tap valid)
    __shared__ float s_w[DCN_PIX][DCN_MAXK][4];      // bilinear weights
    __shared__ float s_m[DCN_PIX][DCN_MAXK];         // modulation mask (1 for DCNv1)
    const int K = p.KH * p.KW;
    const long long npix = (long long)p.B * p.Ho * p.Wo;
    const long long pix0 = (long long)blockIdx.x * DCN_PIX;
    const int cpg = p.C / p.dg;                      // channels per deformable group
    const int g = blockIdx.y;                        // deformable group
    // ---- phase 1: sampling coordinates / weights / mask, once per (pixel, tap) ------------------------------------------
    for (int i = threadIdx.x; i < DCN_PIX * K; i += DCN_THREADS) {
        int pl = i / K, k = i - pl * K;
        long long pix = pix0 + pl;
        int flags = 0, base = 0;
        float w1 = 0.f, w2 = 0.f, w3 = 0.f, w4 = 0.f, m = 1.f;
        if (pix < npix) {
            int wo = (int)(pix % p.Wo); long long r = pix / p.Wo; int ho = (int)(r % p.Ho);
            int kh = k / p.KW, kw = k - kh * p.KW;
            const float* op = p.off + pix * p.off_cs + p.off_co + g * 2 * K + 2 * k;
            float dh = __ldg(op), dw = __ldg(op + 1);
            if (p.msk) {
                m = __ldg(p.msk + pix * p.msk_cs + p.msk_co + g * K + k);
                if (p.mask_sigmoid) m = __fdiv_rn(1.0f, 1.0f + expf(-m));
            }
            float h = (float)(ho * p.stride - p.pad + kh * p.dil) + dh;
            float w = (float)(wo * p.stride - p.pad + kw * p.dil) + dw;
            if (h > -1.f && w > -1.f && h < (float)p.H && w < (float)p.W) {
                int hl = (int)floorf(h), wl = (int)floorf(w);
                float lh = h - (float)hl, lw = w - (float)wl, hh = 1.f - lh, hw = 1.f - lw;
                flags = 16;
                if (hl >= 0 && wl >= 0) flags |= 1;
                if (hl >= 0 && wl + 1 <= p.W - 1) flags |= 2;
                if (hl + 1 <= p.H - 1 && wl >= 0) flags |= 4;
                if (hl + 1 <= p.H - 1 && wl + 1 <= p.W - 1) flags |= 8;
                base = hl * p.W + wl;                 // may be "negative" (hl or wl == -1): those neighbours are masked by flags
                w1 = hh * hw; w2 = hh * lw; w3 = lh * hw; w4 = lh * lw;
            }
        }
        s_base[pl][k][0] = base; s_base[pl][k][1] = flags;
        s_w[pl][k][0] = w1; s_w[pl][k][1] = w2; s_w[pl][k][2] = w3; s_w[pl][k][3] = w4;
        s_m[pl][k] = m;
    }
    __syncthreads();
    // ---- phase 2: gather.  work item = (pixel, tap, channel quad of this deformable group) -----------------------------
    const int cq = cpg / 4;
    const int items = DCN_PIX * K * cq;
    for (int i = threadIdx.x; i < items; i += DCN_THREADS) {
        int q = i % cq; int r = i / cq; int k = r % K; int pl = r / K;
        long long pix = pix0 + pl;
        if (pix >= npix) continue;
        int b = (int)(pix / ((long long)p.Ho * p.Wo));
        int c = g * cpg + 4 * q;
        int flags = s_base[pl][k][1], base = s_base[pl][k][0];
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        if (flags & 16) {
            const float* xb = p.x + ((long long)b * p.H * p.W) * p.x_cs + p.x_co + c;
            float4 v1 = (flags & 1) ? ldg4(xb + (long long)base * p.x_cs) : make_float4(0.f, 0.f, 0.f, 0.f);
            float4 v2 = (flags & 2) ? ldg4(xb + (long long)(base + 1) * p.x_cs) : make_float4(0.f, 0.f, 0.f, 0.f);
            float4 v3 = (flags & 4) ? ldg4(xb + (long long)(base + p.W) * p.x_cs) : make_float4(0.f, 0.f, 0.f, 0.f);
            float4 v4 = (flags & 8) ? ldg4(xb + (long long)(base + p.W + 1) * p.x_cs) : make_float4(0.f, 0.f, 0.f, 0.f);
            float w1 = s_w[pl][k][0], w2 = s_w[pl][k][1], w3 = s_w[pl][k][2], w4 = s_w[pl][k][3];
            // explicit operation order (shared with dcn_fused.cu, whose columns must have the same bits): ((w1 v1 + w2 v2) + w3 v3) + w4 v4 as an fma chain
            acc.x = fmaf(w4, v4.x, fmaf(w3, v3.x, fmaf(w2, v2.x, __fmul_rn(w1, v1.x))));
            acc.y = fmaf(w4, v4.y, fmaf(w3, v3.y, fmaf(w2, v2.y, __fmul_rn(w1, v1.y))));
            acc.z = fmaf(w4, v4.z, fmaf(w3, v3.z, fmaf(w2, v2.z, __fmul_rn(w1, v1.z))));
            acc.w = fmaf(w4, v4.w, fmaf(w3, v3.w, fmaf(w2, v2.w, __fmul_rn(w1, v1.w))));
        }
        float m = s_m[pl][k];
        acc.x = __fmul_rn(acc.x, m); acc.y = __fmul_rn(acc.y, m); acc.z = __fmul_rn(acc.z, m); acc.w = __fmul_rn(acc.w, m);
        long long o = pix * p.col_cs + (p.k_order ? (long long)((c >> 6) * K + k) * 64 + (c & 63) : (long long)k * p.C + c);
        if (p.col) *reinterpret_cast<float4*>(p.col + o) = acc;
        if (p.col_h16_hi) {     // hi = rn16(v), lo = rn16(v - hi): identical to vd3d_split_h16_nhwc on the fp32 columns
            note_fp16_range(amax4(0.f, acc), p.range_flag);
            __half hx = __float2half_rn(acc.x), hy = __float2half_rn(acc.y), hz = __float2half_rn(acc.z), hw = __float2half_rn(acc.w);
            __half2 h01 = __halves2half2(hx, hy), h23 = __halves2half2(hz, hw);
            __half2 l01 = __halves2half2(__float2half_rn(acc.x - __half2float(hx)), __float2half_rn(acc.y - __half2float(hy)));
            __half2 l23 = __halves2half2(__float2half_rn(acc.z - __half2float(hz)), __float2half_rn(acc.w - __half2float(hw)));
            uint2 hv, lv;
            hv.x = *reinterpret_cast<uint32_t*>(&h01); hv.y = *reinterpret_cast<uint32_t*>(&h23);
            lv.x = *reinterpret_cast<uint32_t*>(&l01); lv.y = *reinterpret_cast<uint32_t*>(&l23);
            *reinterpret_cast<uint2*>(p.col_h16_hi + o) = hv;
            *reinterpret_cast<uint2*>(p.col_h16_lo + o) = lv;
        }
        if (p.col_lo) {
            float4 l;
            l.x = acc.x - __uint_as_float(__float_as_uint(acc.x) & 0xFFFFE000u);
            l.y = acc.y - __uint_as_float(__float_as_uint(acc.y) & 0xFFFFE000u);
            l.z = acc.z - __uint_as_float(__float_as_uint(acc.z) & 0xFFFFE000u);
            l.w = acc.w - __uint_as_float(__float_as_uint(acc.w) & 0xFFFFE000u);
            *reinterpret_cast<float4*>(p.col_lo + o) = l;
        }
    }
}

}  // namespace vd3d

using namespace vd3d;

static int deform_im2col_launch(const float* x, int B, int H, int W, int C, int x_cs, int x_co,
                                const float* off, int off_cs, int off_co,
                                const float* msk, int msk_cs, int msk_co, int mask_sigmoid,
                                int KH, int KW, int stride, int pad, int dil, int deform_groups,
                                float* col, float* col_lo, void* col_hi16, void* col_lo16, int col_cs, void* stream, int k_order = 0) {
    VD3D_REQUIRE(x && off && (col || col_hi16), "deform_im2col: null pointer");
    VD3D_REQUIRE(!col_hi16 || col_lo16, "deform_im2col: fp16 planes come in (hi, lo) pairs");
    VD3D_REQUIRE(B > 0 && H > 0 && W > 0 && C > 0 && KH > 0 && KW > 0 && KH * KW <= DCN_MAXK, "deform_im2col: bad shape (<= 49 taps)");
    VD3D_REQUIRE(deform_groups >= 1 && C % deform_groups == 0 && (C / deform_groups) % 4 == 0, "deform_im2col: channels per deformable group must be a multiple of 4");
    VD3D_REQUIRE(x_cs % 4 == 0 && x_co % 4 == 0 && col_cs % 4 == 0 && col_cs >= KH * KW * C, "deform_im2col: pitches/offsets must be multiples of 4");
    DcnParams p;
    p.x = x; p.B = B; p.H = H; p.W = W; p.C = C; p.x_cs = x_cs; p.x_co = x_co;
    p.off = off; p.off_cs = off_cs; p.off_co = off_co; p.msk = msk; p.msk_cs = msk_cs; p.msk_co = msk_co; p.mask_sigmoid = mask_sigmoid;
    p.KH = KH; p.KW = KW; p.stride = stride; p.pad = pad; p.dil = dil; p.dg = deform_groups;
    p.Ho = (H + 2 * pad - (dil * (KH - 1) + 1)) / stride + 1;
    p.Wo = (W + 2 * pad - (dil * (KW - 1) + 1)) / stride + 1;
    VD3D_REQUIRE(p.Ho > 0 && p.Wo > 0, "deform_im2col: empty output");
    p.col = col; p.col_lo = col_lo; p.col_cs = col_cs; p.col_h16_hi = (__half*)col_hi16; p.col_h16_lo = (__half*)col_lo16;
    p.range_flag = col_hi16 ? fp16_range_flag() : nullptr;
    VD3D_REQUIRE(k_order == 0 || (k_order == 1 && C % 64 == 0 && deform_groups == 1), "deform_im2col: the chunk-major column order needs C % 64 == 0 and one deformable group");
    p.k_order = k_order;
    long long npix = (long long)B * p.Ho * p.Wo;
    dim3 grid(cdiv(npix, DCN_PIX), deform_groups);
    deform_im2col_kernel<<<grid, DCN_THREADS, 0, (cudaStream_t)stream>>>(p);
    VD3D_CHECK_LAUNCH("deform_im2col");
    return VD3D_OK;
}

extern "C" int vd3d_deform_im2col_nhwc(const float* x, int B, int H, int W, int C, int x_cs, int x_co,
                                       const float* off, int off_cs, int off_co,
                                       const float* msk, int msk_cs, int msk_co, int mask_sigmoid,
                                       int KH, int KW, int stride, int pad, int dil, int deform_groups,
                                       float* col, float* col_lo, int col_cs, void* stream) {
    VD3D_REQUIRE(col, "deform_im2col: null pointer");
    return deform_im2col_launch(x, B, H, W, C, x_cs, x_co, off, off_cs, off_co, msk, msk_cs, msk_co, mask_sigmoid, KH, KW, stride, pad, dil, deform_groups,
                                col, col_lo, nullptr, nullptr, col_cs, stream);
}

extern "C" int vd3d_deform_im2col_h16(const float* x, int B, int H, int W, int C, int x_cs, int x_co,
                                      const float* off, int off_cs, int off_co,
                                      const float* msk, int msk_cs, int msk_co, int mask_sigmoid,
                                      int KH, int KW, int stride, int pad, int dil, int deform_groups, int k_order,
                                      float* col, void* col_hi16, void* col_lo16, int col_cs, void* stream) {
    VD3D_REQUIRE(col_hi16 && col_lo16, "deform_im2col_h16: null pointer");
    return deform_im2col_launch(x, B, H, W, C, x_cs, x_co, off, off_cs, off_co, msk, msk_cs, msk_co, mask_sigmoid, KH, KW, stride, pad, dil, deform_groups,
                                col, nullptr, col_hi16, col_lo16, col_cs, stream, k_order);
}
