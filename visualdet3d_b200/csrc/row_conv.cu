// Few-channel KHxKW convolutions (the DLA-34 front end: base_layer 7x7 3 -> 16, level0 3x3 16 -> 16, level1 3x3 / 2 16 -> 32 at full image
// resolution, R/networks/backbones/dla.py:246-262) on the Hopper tensor cores (wgmma) as ROW-STRIP kernels: the generalisation of stem_pool.cu
// without the pool.
//
// The input is kept as fp16 (hi, lo) ROW PLANES [B][H][Wp][PC] (PC = 4, 8 or 16 channels = 8, 16 or 32 bytes per pixel, `xoff` >= pad zero pixels
// in front of every row, zeros behind).  For filter row ky the KW * PC operand values of output column m are CONTIGUOUS in the staged image row and
// start S * PC * 2 bytes after those of column m - 1.  A K-major no-swizzle wgmma operand has its core-matrix rows 16 bytes apart, so the
// descriptor (leading byte offset 16, stride byte offset 128) reads operand row r at byte 16 r of the staged row: output column m is operand row
// RS * m with RS = S * PC * 2 / 16 (1, 2 or 4); the rows in between are windows that start inside a pixel: computed and ignored.  A tile is one
// conv row x 128 / RS output columns; nothing is gathered or re-laid-out, and an image row is loaded once per strip (ring of 16 rows, 1-D bulk
// copies, rows outside the image zero-filled by the producer warp).  Weights: KH blocks [N][KS * 16] fp16 hi | lo (k = kx * PC + c, zero beyond
// KW * PC), resident in shared memory.  Three MMAs per K step (A_lo W_hi, A_hi W_lo, A_hi W_hi), promotion chunks of <= 4 filter rows.
// Warps 0..7 = two consumer warpgroups (operand rows 64 w .. 64 w + 63: MMAs, promotion, then the epilogue of the conv row through a staged
// [128][N + 4] shared-memory tile), warp 8 = row producer.
#include "tc_conv.cuh"

namespace vd3d {

constexpr int RC_THREADS = 256 + 32;             // warps: 0..7 = consumers, 8 = row producer
constexpr int RC_RING = 16;                      // staged image rows

struct RcParams {
    const uint8_t* in_hi; const uint8_t* in_lo;  // row planes [B][H][Wp][PC] fp16
    int B, H, Wp, pxb;                           // pxb = bytes per pixel and plane
    int KH, S, P, KS, RS;                        // filter rows, stride, padding, K steps per filter row, operand rows per output column
    int xbyte0;                                  // byte offset inside a padded row of the window of output column 0: (xoff - P) * pxb
    int Ho, Wo;
    int nstrips, nseg, seg_rows, pxs;            // pxs = output columns per strip = 128 / RS
    int rowb;                                    // staged bytes per image row and plane
    int N, w_block;                              // output channels; bytes of one filter-row weight block per plane (N * KS * 32)
    uint32_t w_layout, w_sbo;                    // descriptor layout type / stride byte offset of the weight blocks (SWIZZLE_64B: 4 / 512, SWIZZLE_128B: 2 / 1024)
    float out_scale; const float* bias; int relu;
    float* out; __half* out_hi; __half* out_lo;  // NHWC [B][Ho][out_W][out_cs], image column x at out_xoff + x
    int out_W, out_xoff, out_cs, out_co;
    int* range_flag;
    int dbg;
};

__device__ __forceinline__ void rc_bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes),
                 "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void rc_unit(const RcParams& q, int u, int& b, int& strip, int& y0, int& T) {
    const int seg = u % q.nseg; u /= q.nseg;
    strip = u % q.nstrips; b = u / q.nstrips;
    y0 = seg * q.seg_rows;
    T = min(q.seg_rows, q.Ho - y0);
}

template <int N>
__global__ void __launch_bounds__(RC_THREADS, 1)
row_conv_kernel(const __grid_constant__ CUtensorMap mapWhi, const __grid_constant__ CUtensorMap mapWlo, const RcParams q) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    constexpr int LD = N + 4;
    uint8_t* wsm = smem;                                                       // [KH][hi | lo] weight blocks
    uint8_t* ring = wsm + (((size_t)q.KH * 2 * q.w_block + 1023) & ~(size_t)1023);      // [RC_RING][hi | lo] image rows
    const uint32_t slotb = 2u * (uint32_t)q.rowb;
    float* tile = reinterpret_cast<float*>(ring + (size_t)RC_RING * slotb);   // [128][LD] staged accumulator of one conv row
    uint64_t* bars = reinterpret_cast<uint64_t*>(tile + 128 * LD);
    uint64_t* full = bars;                       // [RC_RING]
    uint64_t* empty = full + RC_RING;            // [RC_RING]  consumers (8 warps) -> producer
    uint64_t* fullW = empty + RC_RING;           // [1]

    const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
    const int units = q.B * q.nstrips * q.nseg;
    const int u0 = (int)blockIdx.x, ustep = (int)gridDim.x;
    const int NCH = q.KH > 4 ? 2 : 1;            // promotion chunks per conv row

    if (threadIdx.x == 0) {
        for (int s = 0; s < RC_RING; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
        mbar_init(fullW, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    pdl_launch_dependents();
    pdl_wait();

    if (warp == 8) {
        // ================= producer: the weights once, then S image rows per conv row =================
        if (elect_one()) {
            mbar_expect_tx(fullW, (uint32_t)q.KH * 2u * (uint32_t)q.w_block);
            for (int ky = 0; ky < q.KH; ++ky) {
                tma_load_2d(wsm + (size_t)ky * 2 * q.w_block, &mapWhi, fullW, ky * q.KS * 16, 0);
                tma_load_2d(wsm + (size_t)ky * 2 * q.w_block + q.w_block, &mapWlo, fullW, ky * q.KS * 16, 0);
            }
        }
        __syncwarp();
        int gl = 0;
        for (int u = u0; u < units; u += ustep) {
            int b, strip, y0, T;
            rc_unit(q, u, b, strip, y0, T);
            const int L = q.S * (T - 1) + q.KH;                     // image rows of the unit
            const int yi0 = q.S * y0 - q.P;
            const size_t xbyte = (size_t)q.xbyte0 + (size_t)strip * 2048;
            for (int l = 0; l < L; ++l, ++gl) {
                const int slot = gl % RC_RING;
                mbar_wait(&empty[slot], ((gl / RC_RING) & 1) ^ 1);
                uint8_t* dst = ring + (size_t)slot * slotb;
                const int yi = yi0 + l;
                const bool inside = yi >= 0 && yi < q.H;
                if (!inside) {                                       // out-of-image row: zeros (the conv's padding)
                    uint4* z = reinterpret_cast<uint4*>(dst);
                    for (int i = lane; i < (int)(slotb / 16); i += 32) z[i] = make_uint4(0u, 0u, 0u, 0u);
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                }
                __syncwarp();
                if (elect_one()) {
                    mbar_expect_tx(&full[slot], inside ? slotb : 0u);
                    if (inside) {
                        const size_t off = ((size_t)b * q.H + yi) * (size_t)q.Wp * q.pxb + xbyte;
                        rc_bulk_g2s(dst, q.in_hi + off, (uint32_t)q.rowb, &full[slot]);
                        rc_bulk_g2s(dst + q.rowb, q.in_lo + off, (uint32_t)q.rowb, &full[slot]);
                    }
                }
                __syncwarp();
            }
        }
    } else {
        // ================= consumer warpgroups: MMAs of operand rows 64 wg .. 64 wg + 63, promotion, epilogue =================
        const int wg = warp >> 2;
        const int qd = warp & 3, half = warp >> 2;
        const int r = qd * 32 + lane;                                  // epilogue: operand row of this thread, columns [half N / 2, +N / 2)
        const float osc = q.out_scale;
        const bool lane_px = (r % q.RS) == 0;
        const int xl = r / q.RS;                                       // output column inside the strip
        auto release = [&](int slot) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[slot]);
        };
        mbar_wait(fullW, 0);
        const uint32_t wbase = smem_u32(wsm), rbase = smem_u32(ring);
        float amax = 0.f;
        float tot[N / 2], c[N / 2];
        int gl = 0;
        for (int u = u0; u < units; u += ustep) {
            int b, strip, y0, T;
            rc_unit(q, u, b, strip, y0, T);
            const int x = strip * q.pxs + xl;
            const bool ok = lane_px && x < q.Wo && !(q.dbg & 16);
            for (int t = 0; t < T; ++t) {
                // conv row t reads local image rows S t .. S t + KH - 1; rows up to S t + KH - S - 1 were waited for by earlier conv rows
                for (int l = (t == 0 ? 0 : q.S * t + q.KH - q.S); l < q.S * t + q.KH; ++l) mbar_wait(&full[(gl + l) % RC_RING], ((gl + l) / RC_RING) & 1);
#pragma unroll
                for (int k = 0; k < N / 2; ++k) tot[k] = 0.f;
                for (int chunk = 0; chunk < NCH; ++chunk) {
                    const int ky0 = chunk * 4, ky1 = (chunk == NCH - 1) ? q.KH : 4;
                    wg_fence();
                    for (int ky = ky0; ky < ky1; ++ky) {
                        const uint32_t ra = rbase + (uint32_t)((gl + q.S * t + ky) % RC_RING) * slotb + (uint32_t)wg * 64u * 16u;
                        const uint32_t wa = wbase + (uint32_t)(ky * 2 * q.w_block);
                        for (int s = 0; s < q.KS; ++s) {
                            const uint64_t dA = make_sdesc_ns(ra + 32u * s, 16u, 128u), dAlo = make_sdesc_ns(ra + q.rowb + 32u * s, 16u, 128u);
                            const uint64_t dB = make_sdesc(wa, q.w_sbo, q.w_layout) + (uint64_t)(2 * s);
                            const uint64_t dBlo = make_sdesc(wa + q.w_block, q.w_sbo, q.w_layout) + (uint64_t)(2 * s);
                            const uint32_t first = (ky == ky0 && s == 0) ? 0u : 1u;
                            if (q.dbg & 1) { wgmma_f16<N>(c, dA, dB, first); continue; }
                            wgmma_f16<N>(c, dAlo, dB, first);
                            wgmma_f16<N>(c, dA, dBlo, 1u);
                            wgmma_f16<N>(c, dA, dB, 1u);
                        }
                    }
                    wg_commit();
                    wg_wait<0>();
                    wg_promote(tot, c);
                }
                for (int l = q.S * t; l < q.S * (t + 1); ++l) release((gl + l) % RC_RING);      // not read by the next conv row
                consumers_sync();                                      // the previous conv row's staged accumulator has been read
                wg_stage<N>(tot, tile, LD, wg, warp, lane);
                consumers_sync();
                if (ok) {
                    const float* acc = tile + r * LD;
                    const long long pix = ((long long)b * q.Ho + (y0 + t)) * q.out_W + q.out_xoff + x;
                    const long long o = pix * q.out_cs + q.out_co;
#pragma unroll
                    for (int k = half * (N / 2); k < (half + 1) * (N / 2); k += 8) {
                        float a[8];
#pragma unroll
                        for (int m = 0; m < 8; m += 4) {
                            const float4 bb = q.bias ? ldg4(q.bias + k + m) : make_float4(0.f, 0.f, 0.f, 0.f);
                            const float4 av = *reinterpret_cast<const float4*>(acc + k + m);
                            a[m] = av.x * osc + bb.x; a[m + 1] = av.y * osc + bb.y;
                            a[m + 2] = av.z * osc + bb.z; a[m + 3] = av.w * osc + bb.w;
                        }
                        if (q.relu) {
#pragma unroll
                            for (int m = 0; m < 8; ++m) a[m] = fmaxf(a[m], 0.f);
                        }
                        if (q.out) {
                            *reinterpret_cast<float4*>(q.out + o + k) = make_float4(a[0], a[1], a[2], a[3]);
                            *reinterpret_cast<float4*>(q.out + o + k + 4) = make_float4(a[4], a[5], a[6], a[7]);
                        }
                        if (q.out_hi) {
#pragma unroll
                            for (int m = 0; m < 8; ++m) amax = fmaxf(amax, fabsf(a[m]));
                            uint2 h0, l0, h1, l1;
                            split4(a, h0, l0);
                            split4(a + 4, h1, l1);
                            *reinterpret_cast<uint4*>(q.out_hi + o + k) = make_uint4(h0.x, h0.y, h1.x, h1.y);
                            *reinterpret_cast<uint4*>(q.out_lo + o + k) = make_uint4(l0.x, l0.y, l1.x, l1.y);
                        }
                    }
                }
            }
            const int L = q.S * (T - 1) + q.KH;
            for (int l = q.S * T; l < L; ++l) release((gl + l) % RC_RING);
            gl += L;
        }
        if (q.out_hi) note_fp16_range(amax, q.range_flag);
    }
}

// NCHW float image -> fp16 (hi, lo) row planes [B][H][Wp][cpad] (cpad = 4 or 8 channels per pixel, channels >= C zero), image column x at xoff + x
__global__ void image_to_h16_rows_c_kernel(const float* __restrict__ in, __half* __restrict__ hi, __half* __restrict__ lo, int C, int H, int W,
                                           long long total, int Wp, int xoff, int cpad, int* __restrict__ range_flag) {
    long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const long long HW = (long long)H * W;
    const long long b = idx / HW, pq = idx - b * HW;
    const int y = (int)(pq / W), x = (int)(pq - (long long)y * W);
    const float* ip = in + b * C * HW + pq;
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float am = 0.f;
    for (int c = 0; c < C; ++c) { v[c] = __ldg(ip + (long long)c * HW); am = fmaxf(am, fabsf(v[c])); }
    note_fp16_range(am, range_flag);
    const long long o = ((b * H + y) * Wp + x + xoff) * cpad;
    for (int c0 = 0; c0 < cpad; c0 += 4) {
        uint2 hv, lv;
        split4(v + c0, hv, lv);
        *reinterpret_cast<uint2*>(hi + o + c0) = hv;
        *reinterpret_cast<uint2*>(lo + o + c0) = lv;
    }
}

}  // namespace vd3d

using namespace vd3d;

extern "C" int vd3d_image_to_h16_rows_c(const float* img, int B, int C, int H, int W, void* hi16, void* lo16, int Wp, int xoff, int cpad, void* stream) {
    VD3D_REQUIRE(img && hi16 && lo16 && B > 0 && C >= 1 && (cpad == 4 || cpad == 8) && C <= cpad && H > 0 && W > 0 && xoff >= 0 && Wp >= W + xoff, "image_to_h16_rows_c: bad args");
    const long long total = (long long)B * H * W;
    image_to_h16_rows_c_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(img, (__half*)hi16, (__half*)lo16, C, H, W, total, Wp, xoff, cpad, fp16_range_flag());
    VD3D_CHECK_LAUNCH("image_to_h16_rows_c");
    return VD3D_OK;
}

// smallest row pitch (pixels) of INPUT planes with `pc` channels per pixel for a KW-wide, stride-S, pad-P row conv over W image columns with `xoff`
// zero pixels in front of every row: the last strip's staged row must stay inside the row
extern "C" int vd3d_row_conv_pitch(int W, int pc, int KW, int S, int P, int xoff) {
    const int pxb = pc * 2;
    if (pxb != 8 && pxb != 16 && pxb != 32) return -1;
    const int RS = S * pxb / 16;
    if (RS < 1 || RS > 4 || S * pxb % 16 != 0 || xoff < P) return -1;
    const int Wo = (W + 2 * P - KW) / S + 1;
    const int pxs = 128 / RS;
    const int nstrips = (Wo + pxs - 1) / pxs;
    const int KS = KW * pxb <= 64 ? 2 : 4;              // K steps (32 bytes) per filter row: 64-byte (SWIZZLE_64B) or 128-byte weight rows
    if (KW * pxb > 128) return -1;
    const int rowb = (127 * 16 + KS * 32 + 15) / 16 * 16;
    const long long bytes = (long long)(xoff - P) * pxb + 2048LL * (nstrips - 1) + rowb;
    int need = (int)((bytes + pxb - 1) / pxb);
    if (need < W + xoff) need = W + xoff;
    return (need + 3) / 4 * 4;
}

// out = act(conv(in) * out_scale + bias): in = row planes [B][H][Wp][pc] (image column x at xoff + x; the buffer is zero outside the image columns),
// weights = [N][KH * KS * 16] fp16 (hi, lo) with k = ky * KS * 16 + kx * pc + c, KS = ceil(KW * pc / 16), N = 16 or 32;
// out = NHWC [B][Ho][out_W][out_cs] (fp32 `out`, may be NULL, and / or fp16 (hi, lo) planes, may be NULL), image column x at out_xoff + x.
extern "C" int vd3d_row_conv(const void* in_hi, const void* in_lo, int B, int H, int W, int Wp, int xoff, int pc, int KH, int KW, int S, int P,
                             const void* w_hi, const void* w_lo, float out_scale, const float* bias, int relu, int N,
                             float* out, void* out_hi16, void* out_lo16, int out_W, int out_xoff, int out_cs, int out_co, void* stream) {
    VD3D_REQUIRE(in_hi && in_lo && w_hi && w_lo && (out || out_hi16), "row_conv: null pointer");
    VD3D_REQUIRE(!out_hi16 == !out_lo16, "row_conv: fp16 output planes come in (hi, lo) pairs");
    VD3D_REQUIRE(N == 16 || N == 32, "row_conv: 16 or 32 output channels (got %d)", N);
    VD3D_REQUIRE(KH >= 1 && KH <= 7 && KW >= 1 && S >= 1 && S <= 2 && P >= 0, "row_conv: KH <= 7, stride 1 or 2");
    VD3D_REQUIRE(vd3d_row_conv_pitch(W, pc, KW, S, P, xoff) > 0 && Wp >= vd3d_row_conv_pitch(W, pc, KW, S, P, xoff) && (Wp * pc * 2) % 16 == 0,
                 "row_conv: row pitch %d < vd3d_row_conv_pitch() = %d (or unsupported channel count / stride)", Wp, vd3d_row_conv_pitch(W, pc, KW, S, P, xoff));
    VD3D_REQUIRE(out_cs % 8 == 0 && out_co % 8 == 0, "row_conv: output pitch / offset must be multiples of 8 channels");
    VD3D_REQUIRE((((uintptr_t)in_hi | (uintptr_t)in_lo | (uintptr_t)w_hi | (uintptr_t)w_lo | (uintptr_t)out | (uintptr_t)out_hi16 | (uintptr_t)out_lo16 | (uintptr_t)bias) & 15) == 0,
                 "row_conv: pointers must be 16-byte aligned");
    RcParams q;
    memset(&q, 0, sizeof(q));
    q.in_hi = (const uint8_t*)in_hi; q.in_lo = (const uint8_t*)in_lo; q.B = B; q.H = H; q.Wp = Wp; q.pxb = pc * 2;
    q.KH = KH; q.S = S; q.P = P; q.KS = KW * q.pxb <= 64 ? 2 : 4; q.RS = S * q.pxb / 16;
    VD3D_REQUIRE(KH >= S, "row_conv: KH >= stride");
    VD3D_REQUIRE(((xoff - P) * q.pxb) % 16 == 0, "row_conv: (xoff - pad) pixels must be a multiple of 16 bytes");
    q.xbyte0 = (xoff - P) * q.pxb;
    q.Ho = (H + 2 * P - KH) / S + 1; q.Wo = (W + 2 * P - KW) / S + 1;
    VD3D_REQUIRE(q.Ho > 0 && q.Wo > 0, "row_conv: empty output");
    VD3D_REQUIRE(out_W >= q.Wo + out_xoff, "row_conv: output row pitch too small");
    q.pxs = 128 / q.RS; q.nstrips = (q.Wo + q.pxs - 1) / q.pxs;
    q.rowb = (127 * 16 + q.KS * 32 + 15) / 16 * 16;
    {
        long long best = -1;
        for (int n = 1; n <= 32 && n <= q.Ho; ++n) {
            const int rows = (q.Ho + n - 1) / n;
            const int nseg = (q.Ho + rows - 1) / rows;
            const long long units = (long long)B * q.nstrips * nseg;
            const long long cost = ((units + 2 * kNumSMs - 1) / (2 * kNumSMs)) * (rows + KH);
            if (best < 0 || cost < best) { best = cost; q.nseg = nseg; q.seg_rows = rows; }
        }
    }
    q.N = N; q.w_block = N * q.KS * 32;
    q.w_layout = q.KS == 4 ? 2u : 4u; q.w_sbo = q.KS == 4 ? 1024u : 512u;
    q.out_scale = out_scale; q.bias = bias; q.relu = relu;
    q.out = out; q.out_hi = (__half*)out_hi16; q.out_lo = (__half*)out_lo16; q.out_W = out_W; q.out_xoff = out_xoff; q.out_cs = out_cs; q.out_co = out_co;
    q.range_flag = out_hi16 ? fp16_range_flag() : nullptr;
    { const char* e = getenv("VD3D_TC_DEBUG"); q.dbg = e ? atoi(e) : 0; }
    CUtensorMap mWhi, mWlo;
    int rc;
    if ((rc = make_map_wgt(&mWhi, w_hi, N, KH * q.KS * 16, N, 2, q.KS * 32))) return rc;
    if ((rc = make_map_wgt(&mWlo, w_lo, N, KH * q.KS * 16, N, 2, q.KS * 32))) return rc;
    const size_t wbytes = ((size_t)KH * 2 * q.w_block + 1023) & ~(size_t)1023;
    const size_t smem = wbytes + (size_t)RC_RING * 2 * q.rowb + (size_t)128 * (N + 4) * sizeof(float) + (2 * RC_RING + 1) * sizeof(uint64_t) + 1024;
    static bool attr_set = false;
    if (!attr_set) {
        VD3D_CUDA(cudaFuncSetAttribute(row_conv_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        VD3D_CUDA(cudaFuncSetAttribute(row_conv_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        attr_set = true;
    }
    VD3D_REQUIRE(smem <= 227 * 1024, "row_conv: shared-memory budget exceeded");
    const int units = B * q.nstrips * q.nseg;
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    const int slots = smem <= 110 * 1024 ? 2 * kNumSMs : kNumSMs;        // two CTAs per SM when they fit: one hides the other's per-row hand-offs
    cfg.gridDim = dim3((unsigned)(units < slots ? units : slots)); cfg.blockDim = dim3(RC_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = (cudaStream_t)stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = pdl_enabled() ? 1 : 0;
    const cudaError_t le = N == 16 ? cudaLaunchKernelEx(&cfg, row_conv_kernel<16>, mWhi, mWlo, q) : cudaLaunchKernelEx(&cfg, row_conv_kernel<32>, mWhi, mWlo, q);
    if (le != cudaSuccess) { set_error("row_conv: launch failed: %s", cudaGetErrorString(le)); return VD3D_ECUDA; }
    VD3D_CHECK_LAUNCH("row_conv");
    return VD3D_OK;
}
