// ResNet stem as ONE persistent wgmma kernel: conv 7x7 / stride 2 / pad 3 (<= 4 -> 64 channels) + folded BN + ReLU + MaxPool2d(3, 2, 1)
// (R/networks/backbones/resnet.py:120-122,186-189), with NO im2col and no window re-reads from L2.
//
// conv2d_tcp_kernel's stem path presents the image to TMA as a virtual [B][H][Wo][32] tensor with overlapping windows: every tile loads its
// 7 x 128 windows again (3.1 GB of L2 -> SM traffic per batch-16 launch at 384 x 1280), which is what bounds it.
// Here the overlap is expressed in the wgmma shared-memory descriptor instead:
//   * a tile is ONE conv output row x 128 output columns.  For filter row ky the 32 operand values of output column m (8 pixels x 4 channels
//     of the fp16 row planes, pixel 2m .. 2m + 7 of the padded row) start 16 bytes after those of column m - 1.  A K-major, NO-swizzle operand
//     has its 8-row core matrices at a 16-byte row pitch, so with leading byte offset 16 (next 16-byte K chunk) and stride byte offset 128
//     (next 8 rows) the descriptor walks exactly these overlapping windows in the staged image row: A(m, chunk c) = row bytes [16 (m + c), +16).
//     One staged image row (2112 B per plane) is the A operand of all 128 columns; nothing is copied or re-laid-out.
//   * a CTA walks DOWN a strip of 128 conv columns: consecutive conv rows share 5 of their 7 image rows, so the producer streams two new
//     image rows per conv row (1-D bulk copies into a ring of 8 row pairs; out-of-image rows are zero-filled by the producer warp).
//     The weights (7 filter rows x [64][32] fp16 hi | lo, 56 KB) are loaded once per CTA.
//   * warps 0..7 = two consumer warpgroups (strip columns 64 w .. 64 w + 63): the MMAs of a conv row, the promotion of its two chunks, and
//     the epilogue on the accumulator staged in shared memory ([128][68] fp32); warp 8 = producer.
//   * the max-pool happens in registers: thread (column x) keeps the running maximum of its column over the conv rows of the open pooled row;
//     after every second conv row the horizontal 3-max of these column maxima (neighbour columns by warp shuffle, the one column across a warp
//     boundary through 2 KB of shared memory) is the pooled row, and it is written.  Strips overlap by 2 conv columns (63 pooled columns per 128-column strip) and row segments by one conv row, so every
//     3 x 3 window is complete inside one CTA: no atomics, no border pre-zeroing, deterministic.
//   * the pooled tensor is written as the fp16 (hi, lo) planes layer 1 reads (and as fp32 only when asked): the separate max-pool kernel,
//     split kernel and the 126 MB stem output of the unfused path do not exist.
// Accumulation order = conv2d_tcp_kernel's stem path (filter rows 0..3 | 4..6 as the two promotion chunks, two K steps per filter row, three
// MMAs A_lo W_hi, A_hi W_lo, A_hi W_hi per K step), so the result equals the two-kernel path bit for bit (tests/test_ops_gpu.py).
#include "tc_conv.cuh"

namespace vd3d {

constexpr int SP_THREADS = 256 + 32;             // warps: 0..7 = consumers (MMAs, promotion, epilogue), 8 = image-row producer
constexpr int SP_KH = 7, SP_STRIDE = 2, SP_PAD = 3;
constexpr int SP_XOFF = 5;                       // zero pixels in front of every row of the planes (pad 3 + 2: column -1 of strip 0 stays in the row)
constexpr int SP_ROWB = 2112;                    // staged bytes per image row and plane: 264 pixels x 4 channels x fp16
constexpr int SP_ROW = 2 * SP_ROWB;              // hi | lo
constexpr int SP_PAIRS = 8;                      // ring of row pairs
constexpr int SP_PAIR = 2 * SP_ROW;              // 8448 B
constexpr int SP_CENTERS = 63;                   // pooled columns per strip (conv columns 126 t - 1 .. 126 t + 126)
constexpr int SP_WROW = 2 * 64 * 64;             // weights of one filter row: [hi | lo][64 cout][32 k] fp16, SWIZZLE_64B
constexpr int SP_LD = 68;                        // floats per staged accumulator row (64 + 4: conflict-free float4 rows)

struct SpParams {
    const __half* in_hi; const __half* in_lo;    // [B][H][Wp][4]
    int B, H, W, Wp;
    int Ho, Wo, Hq, Wq;                           // conv output, pooled output
    int nstrips, nseg, seg_rows;                  // strips per image row, row segments per strip, pooled rows per segment
    float out_scale; const float* bias;
    float* out; __half* out_hi; __half* out_lo;   // pooled NHWC tensor: fp32 (optional) and / or fp16 (hi, lo) planes (optional)
    int out_cs, out_co;
    int* range_flag;
    int dbg;
};

__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes),
                 "r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ void sp_unit(const SpParams& q, int u, int& b, int& strip, int& i0, int& nrows) {
    const int seg = u % q.nseg; u /= q.nseg;
    strip = u % q.nstrips; b = u / q.nstrips;
    i0 = seg * q.seg_rows;
    nrows = min(q.seg_rows, q.Hq - i0);           // pooled rows of this unit (>= 1 by construction of nseg)
}

__global__ void __launch_bounds__(SP_THREADS, 1)
stem_pool_kernel(const __grid_constant__ CUtensorMap mapWhi, const __grid_constant__ CUtensorMap mapWlo, const SpParams q) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t* wsm = smem;                                          // [7][hi | lo] weights, 1024-byte aligned blocks
    uint8_t* ring = wsm + (size_t)SP_KH * SP_WROW;                // [SP_PAIRS][2 rows][hi | lo]
    float* edge = reinterpret_cast<float*>(ring + (size_t)SP_PAIRS * SP_PAIR);     // [2 parities][2 halves][4 quadrants][32]
    float* stage = edge + 2 * 2 * 4 * 32;                         // [128][SP_LD] staged accumulator of one conv row
    uint64_t* bars = reinterpret_cast<uint64_t*>(stage + 128 * SP_LD);
    uint64_t* full = bars;                       // [SP_PAIRS] producer -> consumers
    uint64_t* empty = full + SP_PAIRS;           // [SP_PAIRS] consumers (8 warps) -> producer
    uint64_t* fullW = empty + SP_PAIRS;          // [1]

    const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
    const int units = q.B * q.nstrips * q.nseg;
    const int u0 = (int)blockIdx.x, ustep = (int)gridDim.x;

    if (threadIdx.x == 0) {
        for (int s = 0; s < SP_PAIRS; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
        mbar_init(fullW, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    pdl_launch_dependents();
    pdl_wait();

    if (warp == 8) {
        // ================= producer: the weights once, then two image rows per conv row =================
        if (elect_one()) {
            mbar_expect_tx(fullW, (uint32_t)SP_KH * SP_WROW);
            for (int ky = 0; ky < SP_KH; ++ky) {
                tma_load_2d(wsm + (size_t)ky * SP_WROW, &mapWhi, fullW, ky * 32, 0);
                tma_load_2d(wsm + (size_t)ky * SP_WROW + SP_WROW / 2, &mapWlo, fullW, ky * 32, 0);
            }
        }
        __syncwarp();
        int gq = 0;
        for (int u = u0; u < units; u += ustep) {
            int b, strip, i0, nrows;
            sp_unit(q, u, b, strip, i0, nrows);
            const int T = 2 * nrows + 1;
            const int yi0 = 4 * i0 - 5;                            // image row of local row 0 (= 2 * (2 i0 - 1) - 3)
            const size_t xbyte = (size_t)strip * (126 * 16);       // byte offset of the strip inside a padded row
            for (int pq = 0; pq < T + 3; ++pq, ++gq) {
                const int slot = gq % SP_PAIRS;
                mbar_wait(&empty[slot], ((gq / SP_PAIRS) & 1) ^ 1);
                uint8_t* dst = ring + (size_t)slot * SP_PAIR;
                uint32_t tx = 0;
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const int yi = yi0 + 2 * pq + r;
                    if (yi >= 0 && yi < q.H) tx += (uint32_t)SP_ROW;
                    else {                                         // out-of-image row: zeros (the conv's padding)
                        uint4* z = reinterpret_cast<uint4*>(dst + (size_t)r * SP_ROW);
                        for (int i = lane; i < SP_ROW / 16; i += 32) z[i] = make_uint4(0u, 0u, 0u, 0u);
                    }
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                __syncwarp();
                if (elect_one()) {
                    mbar_expect_tx(&full[slot], tx);
#pragma unroll
                    for (int r = 0; r < 2; ++r) {
                        const int yi = yi0 + 2 * pq + r;
                        if (yi >= 0 && yi < q.H) {
                            const size_t off = (((size_t)b * q.H + yi) * q.Wp) * 8 + xbyte;
                            bulk_g2s(dst + (size_t)r * SP_ROW, reinterpret_cast<const uint8_t*>(q.in_hi) + off, SP_ROWB, &full[slot]);
                            bulk_g2s(dst + (size_t)r * SP_ROW + SP_ROWB, reinterpret_cast<const uint8_t*>(q.in_lo) + off, SP_ROWB, &full[slot]);
                        }
                    }
                }
                __syncwarp();
            }
        }
    } else {
        // ================= consumer warpgroups: MMAs of strip columns 64 wg .. 64 wg + 63, promotion, bias / ReLU, 3 x 3 / stride-2 max in registers =================
        const int wg = warp >> 2;
        const int e = warp, qd = warp & 3, half = e >> 2;
        const int x = qd * 32 + lane;                                  // epilogue: conv column inside the strip
        const float osc = q.out_scale;
        const int cb = half * 32;
        auto release = [&](int slot) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[slot]);
        };
        mbar_wait(fullW, 0);
        const uint32_t wbase = smem_u32(wsm), rbase = smem_u32(ring);
        float amax = 0.f;
        float tot[32], c[32];
        int gq = 0, tile = 0;
        for (int u = u0; u < units; u += ustep) {
            int b, strip, i0, nrows;
            sp_unit(q, u, b, strip, i0, nrows);
            const int T = 2 * nrows + 1;
            const int cc0 = 126 * strip - 1 + x;                       // conv column
            const bool col_ok = cc0 >= 0 && cc0 < q.Wo;
            const int jl = (x - 1) >> 1;                               // pooled column inside the strip (x odd)
            const int j = SP_CENTERS * strip + jl;
            const bool centre = (x & 1) && jl < SP_CENTERS && j < q.Wq;
            // run[k] = column-wise maximum of the conv rows of the pooled row that is open (vertical max first: the horizontal 3-max, its
            // shuffles and the cross-warp exchange are then needed only once per pooled row, on the maximum of the three conv rows)
            float run[32];
#pragma unroll
            for (int k = 0; k < 32; ++k) run[k] = 0.f;
            for (int t = 0; t < T; ++t) {
                // image rows of conv row t: local rows 2t .. 2t + 6 = pairs t .. t + 3
                for (int pq = (t == 0 ? 0 : t + 3); pq <= t + 3; ++pq) mbar_wait(&full[(gq + pq) % SP_PAIRS], ((gq + pq) / SP_PAIRS) & 1);
#pragma unroll
                for (int k = 0; k < 32; ++k) tot[k] = 0.f;
#pragma unroll 1
                for (int chunk = 0; chunk < 2; ++chunk) {
                    const int ky0 = chunk * 4, ky1 = chunk ? SP_KH : 4;
                    wg_fence();
                    for (int ky = ky0; ky < ky1; ++ky) {
                        const int l = 2 * t + ky;                                        // local image row
                        const uint32_t ra = rbase + (uint32_t)(((gq + (l >> 1)) % SP_PAIRS) * SP_PAIR + (l & 1) * SP_ROW) + (uint32_t)wg * 64u * 16u;
                        const uint32_t wa = wbase + (uint32_t)(ky * SP_WROW);
#pragma unroll
                        for (int s = 0; s < 2; ++s) {
                            const uint64_t dA = make_sdesc_ns(ra + 32u * s, 16u, 128u), dAlo = make_sdesc_ns(ra + SP_ROWB + 32u * s, 16u, 128u);
                            const uint64_t dB = make_sdesc(wa, 512u, 4u) + (uint64_t)(2 * s), dBlo = make_sdesc(wa + SP_WROW / 2, 512u, 4u) + (uint64_t)(2 * s);
                            const uint32_t first = (ky == ky0 && s == 0) ? 0u : 1u;
                            if (q.dbg & 1) { wgmma_f16<64>(c, dA, dB, first); continue; }
                            wgmma_f16<64>(c, dAlo, dB, first);
                            wgmma_f16<64>(c, dA, dBlo, 1u);
                            wgmma_f16<64>(c, dA, dB, 1u);
                        }
                    }
                    wg_commit();
                    wg_wait<0>();
                    wg_promote(tot, c);
                }
                release((gq + t) % SP_PAIRS);                                    // rows 2t, 2t + 1 are not read again
                consumers_sync();                                                // the previous conv row's staged accumulator has been read
                wg_stage<64>(tot, stage, SP_LD, wg, warp, lane);
                consumers_sync();
                float acc[32];
                {
                    const float* sp = stage + x * SP_LD + cb;
#pragma unroll
                    for (int k = 0; k < 32; k += 4) {
                        const float4 v = *reinterpret_cast<const float4*>(sp + k);
                        acc[k] = v.x; acc[k + 1] = v.y; acc[k + 2] = v.z; acc[k + 3] = v.w;
                    }
                }
                const int y = 2 * i0 - 1 + t;                          // conv row
                const bool ok = col_ok && y >= 0 && y < q.Ho;
#pragma unroll
                for (int k = 0; k < 32; k += 4) {
                    const float4 bb = q.bias ? ldg4(q.bias + cb + k) : make_float4(0.f, 0.f, 0.f, 0.f);
                    acc[k] = ok ? fmaxf(acc[k] * osc + bb.x, 0.f) : 0.f;
                    acc[k + 1] = ok ? fmaxf(acc[k + 1] * osc + bb.y, 0.f) : 0.f;
                    acc[k + 2] = ok ? fmaxf(acc[k + 2] * osc + bb.z, 0.f) : 0.f;
                    acc[k + 3] = ok ? fmaxf(acc[k + 3] * osc + bb.w, 0.f) : 0.f;
                }
                if (t == 0) {
#pragma unroll
                    for (int k = 0; k < 32; ++k) run[k] = acc[k];
                } else if (t & 1) {
#pragma unroll
                    for (int k = 0; k < 32; ++k) run[k] = fmaxf(run[k], acc[k]);
                } else {
                    // conv row 2i + 1 closes pooled row i = i0 + t / 2 - 1: column maxima of its three conv rows, then the horizontal 3-max
                    const int i = i0 + (t >> 1) - 1;
#pragma unroll
                    for (int k = 0; k < 32; ++k) run[k] = fmaxf(run[k], acc[k]);
                    float* ed = edge + (((tile & 1) * 2 + half) * 4) * 32;
                    ++tile;
                    if (lane == 0) {                                       // column 32 (qd + 1) of the strip is lane 31's right neighbour
#pragma unroll
                        for (int k = 0; k < 32; k += 4) *reinterpret_cast<float4*>(ed + qd * 32 + k) = make_float4(run[k], run[k + 1], run[k + 2], run[k + 3]);
                    }
                    asm volatile("bar.sync 1, 256;" ::: "memory");
                    const bool last_lane = lane == 31;
                    const float* en = ed + ((qd + 1) & 3) * 32;
                    const bool wrap = qd == 3;                             // column 128 does not exist (and column 127 is no centre)
                    const long long pix = ((long long)b * q.Hq + i) * q.Wq + j;
                    const long long o = pix * q.out_cs + q.out_co + cb;
                    const bool wr = centre && !(q.dbg & 16);
#pragma unroll
                    for (int k = 0; k < 32; k += 8) {
                        float a[8];
#pragma unroll
                        for (int m = 0; m < 8; ++m) {
                            const float lf = __shfl_up_sync(0xffffffffu, run[k + m], 1);      // (lane 0 gets its own value back: lane 0 is never a centre)
                            float rt = __shfl_down_sync(0xffffffffu, run[k + m], 1);
                            if (last_lane) rt = wrap ? 0.f : en[k + m];
                            a[m] = fmaxf(fmaxf(lf, run[k + m]), rt);
                        }
                        if (wr) {
#pragma unroll
                            for (int m = 0; m < 8; ++m) amax = fmaxf(amax, a[m]);
                            if (q.out) {
                                *reinterpret_cast<float4*>(q.out + o + k) = make_float4(a[0], a[1], a[2], a[3]);
                                *reinterpret_cast<float4*>(q.out + o + k + 4) = make_float4(a[4], a[5], a[6], a[7]);
                            }
                            if (q.out_hi) {
                                uint2 h0, l0, h1, l1;
                                split4(a, h0, l0);
                                split4(a + 4, h1, l1);
                                *reinterpret_cast<uint4*>(q.out_hi + o + k) = make_uint4(h0.x, h0.y, h1.x, h1.y);
                                *reinterpret_cast<uint4*>(q.out_lo + o + k) = make_uint4(l0.x, l0.y, l1.x, l1.y);
                            }
                        }
                    }
#pragma unroll
                    for (int k = 0; k < 32; ++k) run[k] = acc[k];          // conv row 2i + 1 is also the first row of pooled row i + 1
                }
            }
            for (int pq = T; pq < T + 3; ++pq) release((gq + pq) % SP_PAIRS);
            gq += T + 3;
        }
        if (q.out_hi) note_fp16_range(amax, q.range_flag);
    }
}

}  // namespace vd3d

using namespace vd3d;

// padded row pitch (pixels) of the fp16 row planes the fused stem reads: SP_XOFF zero pixels, the image, zeros up to the end of the last strip
extern "C" int vd3d_stem_pool_row_pitch(int W) {
    const int Wo = (W + 2 * SP_PAD - SP_KH) / SP_STRIDE + 1;
    const int Wq = (Wo + 2 - 3) / 2 + 1;
    const int nstrips = (Wq + SP_CENTERS - 1) / SP_CENTERS;
    int need = 252 * (nstrips - 1) + 264;
    if (need < W + SP_XOFF) need = W + SP_XOFF;
    return (need + 1) / 2 * 2;
}
extern "C" int vd3d_stem_pool_xoff(void) { return SP_XOFF; }

// conv 7x7 / 2 / 3 (Cin <= 4 -> 64) + bias (folded BN) + ReLU + MaxPool2d(3, 2, 1): image as fp16 (hi, lo) row planes [B][H][Wp][4]
// (vd3d_image_to_h16_rows with xoff = vd3d_stem_pool_xoff(), Wp = vd3d_stem_pool_row_pitch(W)), weights = the [64][7 * 32] fp16 (hi, lo)
// matrices of the 32-element-window stem (k = ky * 32 + kx * 4 + c).  Output: pooled NHWC tensor as fp32 (`out`, may be NULL) and / or fp16
// (hi, lo) planes (may be NULL), pitch out_cs channels.
extern "C" int vd3d_stem_pool_fused(const void* in_hi, const void* in_lo, int B, int H, int W, int Wp, const void* w_hi, const void* w_lo, float out_scale,
                                    const float* bias, float* out, void* out_hi16, void* out_lo16, int out_cs, int out_co, void* stream) {
    VD3D_REQUIRE(in_hi && in_lo && w_hi && w_lo && (out || out_hi16), "stem_pool_fused: null pointer");
    VD3D_REQUIRE(B > 0 && H >= SP_KH - 2 * SP_PAD && W >= 2, "stem_pool_fused: bad image size");
    VD3D_REQUIRE(Wp == vd3d_stem_pool_row_pitch(W), "stem_pool_fused: row pitch %d != vd3d_stem_pool_row_pitch() = %d", Wp, vd3d_stem_pool_row_pitch(W));
    VD3D_REQUIRE(!out_hi16 == !out_lo16, "stem_pool_fused: fp16 output planes come in (hi, lo) pairs");
    VD3D_REQUIRE(out_cs % 8 == 0 && out_co % 8 == 0, "stem_pool_fused: output pitch / offset must be multiples of 8 channels");
    VD3D_REQUIRE((((uintptr_t)in_hi | (uintptr_t)in_lo | (uintptr_t)w_hi | (uintptr_t)w_lo | (uintptr_t)out | (uintptr_t)out_hi16 | (uintptr_t)out_lo16) & 15) == 0,
                 "stem_pool_fused: pointers must be 16-byte aligned");
    SpParams q;
    memset(&q, 0, sizeof(q));
    q.in_hi = (const __half*)in_hi; q.in_lo = (const __half*)in_lo; q.B = B; q.H = H; q.W = W; q.Wp = Wp;
    q.Ho = (H + 2 * SP_PAD - SP_KH) / SP_STRIDE + 1; q.Wo = (W + 2 * SP_PAD - SP_KH) / SP_STRIDE + 1;
    VD3D_REQUIRE(q.Ho > 0 && q.Wo > 0, "stem_pool_fused: empty output");
    q.Hq = (q.Ho + 2 - 3) / 2 + 1; q.Wq = (q.Wo + 2 - 3) / 2 + 1;
    q.nstrips = (q.Wq + SP_CENTERS - 1) / SP_CENTERS;
    {
        // row segments per strip: minimise rounds x conv rows per unit (every unit recomputes one conv row of its upper neighbour)
        long long best = -1;
        int best_n = 1;
        for (int n = 1; n <= 16 && n <= q.Hq; ++n) {
            const int rows = (q.Hq + n - 1) / n;
            const int nseg = (q.Hq + rows - 1) / rows;
            const long long units = (long long)B * q.nstrips * nseg;
            const long long cost = ((units + kNumSMs - 1) / kNumSMs) * (2 * rows + 1);
            if (best < 0 || cost < best) { best = cost; best_n = nseg; q.seg_rows = rows; }
        }
        q.nseg = best_n;
    }
    q.out_scale = out_scale; q.bias = bias; q.out = out; q.out_hi = (__half*)out_hi16; q.out_lo = (__half*)out_lo16; q.out_cs = out_cs; q.out_co = out_co;
    q.range_flag = out_hi16 ? fp16_range_flag() : nullptr;
    { const char* e = getenv("VD3D_TC_DEBUG"); q.dbg = e ? atoi(e) : 0; }
    CUtensorMap mWhi, mWlo;
    int rc;
    if ((rc = make_map_wgt(&mWhi, w_hi, 64, SP_KH * 32, 64, 2, 64))) return rc;
    if ((rc = make_map_wgt(&mWlo, w_lo, 64, SP_KH * 32, 64, 2, 64))) return rc;
    const size_t smem = (size_t)SP_KH * SP_WROW + (size_t)SP_PAIRS * SP_PAIR + (2 * 2 * 4 * 32 + 128 * SP_LD) * sizeof(float) + (2 * SP_PAIRS + 1) * sizeof(uint64_t) + 1024;
    static bool attr_set = false;
    if (!attr_set) {
        VD3D_CUDA(cudaFuncSetAttribute(stem_pool_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_set = true;
    }
    const int units = B * q.nstrips * q.nseg;
    const int grid = units < kNumSMs ? units : kNumSMs;
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3((unsigned)grid); cfg.blockDim = dim3(SP_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = (cudaStream_t)stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = pdl_enabled() ? 1 : 0;
    const cudaError_t le = cudaLaunchKernelEx(&cfg, stem_pool_kernel, mWhi, mWlo, q);
    if (le != cudaSuccess) { set_error("stem_pool_fused: launch failed: %s", cudaGetErrorString(le)); return VD3D_ECUDA; }
    VD3D_CHECK_LAUNCH("stem_pool_fused");
    return VD3D_OK;
}
