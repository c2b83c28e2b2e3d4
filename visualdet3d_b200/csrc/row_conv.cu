// Few-channel convolutions on the Hopper tensor cores (wgmma) as ROW-STRIP kernels, one core for two kernels:
//   * row_conv_kernel: KHxKW conv + bias [+ ReLU], the DLA-34 front end (base_layer 7x7 3 -> 16, level0 3x3 16 -> 16, level1 3x3 / 2 16 -> 32
//     at full image resolution, R/networks/backbones/dla.py:246-262);
//   * stem_pool_kernel: the ResNet stem, conv 7x7 / 2 / 3 (<= 4 -> 64 channels) + folded BN + ReLU + MaxPool2d(3, 2, 1)
//     (R/networks/backbones/resnet.py:120-122,186-189), with no im2col and no window re-reads from L2.
//
// The input is kept as fp16 (hi, lo) ROW PLANES [B][H][Wp][PC] (PC = 4, 8 or 16 channels = 8, 16 or 32 bytes per pixel, zero pixels in front of
// and behind every row).  For filter row ky the KW * PC operand values of output column m are CONTIGUOUS in the staged image row and start
// S * PC * 2 bytes after those of column m - 1.  A K-major no-swizzle wgmma operand has its core-matrix rows 16 bytes apart, so the descriptor
// (leading byte offset 16, stride byte offset 128) reads operand row r at byte 16 r of the staged row: output column m is operand row RS * m with
// RS = S * PC * 2 / 16 (1, 2 or 4); the rows in between are windows that start inside a pixel: computed and ignored.  One staged image row is
// the A operand of all 128 operand rows of a strip; nothing is gathered or re-laid-out.
//   * a unit is one strip of 128 operand rows x T consecutive conv rows of one image.  The CTA walks DOWN the strip: consecutive conv rows
//     share KH - S image rows, so the producer streams S new image rows per conv row into a ring of 16 rows (1-D bulk copies; rows outside the
//     image zero-filled by the producer warp).  The KH filter-row weight blocks [N][KS * 16] fp16 hi | lo (k = kx * PC + c, zero beyond
//     KW * PC) are loaded once per CTA.
//   * warps 0..7 = two consumer warpgroups (operand rows 64 w .. 64 w + 63): per conv row the MMAs of the KH filter rows (KS K steps per filter
//     row, three products A_lo W_hi, A_hi W_lo, A_hi W_hi per K step, promotion chunks of <= 4 filter rows; through wg_tile_kloop, or as one
//     commit group per chunk when KH is a compile-time constant), then the conv row staged as a [128][N + 4] fp32 tile for the kernel's
//     epilogue; warp 8 = row producer.
// The kernels differ in their unit mapping and their epilogue only:
//   * row_conv_kernel: units are conv-row segments, strips 128 / RS output columns apart; bias / ReLU output as fp32 and / or planes.
//   * stem_pool_kernel (PC = 4, RS = 1, N = 64, KS = 2): strips of 128 conv columns starting 126 apart at conv column -1, units of pooled-row
//     segments whose conv rows overlap the upper neighbour's by one, so every 3 x 3 window is complete inside one CTA: no atomics, no border
//     pre-zeroing, deterministic.  The max-pool happens in registers: a thread (conv column) keeps the running maximum of its column over the
//     conv rows of the open pooled row; after every second conv row the horizontal 3-max of these column maxima (neighbour columns by warp
//     shuffle, the one column across a warp boundary through 2 KB of shared memory) is the pooled row, written as the fp16 (hi, lo) planes
//     layer 1 reads (and as fp32 only when asked).  Its accumulation order is conv2d_tcp_kernel's stem path (filter rows 0..3 | 4..6 as the
//     two promotion chunks), so it equals the two-kernel path bit for bit (tests/test_ops_gpu.py).
#include "tc_conv.cuh"

namespace vd3d {

constexpr int RS_THREADS = 256 + 32;             // warps: 0..7 = consumers, 8 = row producer
constexpr int RS_RING = 16;                      // staged image rows
constexpr int RS_CHUNK = 4;                      // filter rows per promotion chunk

struct RsParams {
    const uint8_t* in_hi; const uint8_t* in_lo;  // row planes [B][H][Wp][PC] fp16
    int B, H, Wp, pxb;                           // pxb = bytes per pixel and plane
    int KH, S, P, KS, RS;                        // filter rows, stride, padding, K steps per filter row, operand rows per output column
    int xbyte0, strip_bytes;                     // byte offset inside a padded row of strip 0's first window, byte step from strip to strip
    int Ho, Wo, Hq, Wq;                          // conv output; pooled output (stem_pool_kernel)
    int nstrips, nseg, seg_rows, pxs;            // strips per image row, row segments per strip, rows per segment, output columns per strip
    int rowb;                                    // staged bytes per image row and plane
    int w_block;                                 // bytes of one filter-row weight block per plane (N * KS * 32)
    float out_scale; const float* bias; int relu;
    float* out; __half* out_hi; __half* out_lo;  // NHWC output: fp32 (may be NULL) and / or fp16 (hi, lo) planes (may be NULL), pitch out_cs
    int out_W, out_xoff, out_cs, out_co;         // row_conv_kernel: [B][Ho][out_W][out_cs], image column x at out_xoff + x
    int* range_flag;
    int dbg;                                     // VD3D_TC_DEBUG (timing experiments, results are wrong): bit 0 = one MMA per K step, bit 4 = no output stores
};

struct RsUnit { int b, strip, y0, T; };          // image, strip, conv rows y0 .. y0 + T - 1

// unit u -> image, strip and the segment [first, first + count) of the `rows` rows (conv or pooled) a kernel splits into q.nseg segments
__device__ __forceinline__ void rs_segment(const RsParams& q, int u, int rows, int& b, int& strip, int& first, int& count) {
    const int seg = u % q.nseg; u /= q.nseg;
    strip = u % q.nstrips; b = u / q.nstrips;
    first = seg * q.seg_rows;
    count = min(q.seg_rows, rows - first);
}

// The core.  Epi: the kernel's unit mapping (static unit(q, u) -> RsUnit) and epilogue (begin(unit), row(unit, t, staged conv row t), finish()),
// with Epi::kExtraBytes of shared memory of its own.  KH_FIXED > 0: the filter-row count is a compile-time constant, and each promotion chunk's
// MMAs are issued as one straight-line commit group (the K walk is then fully unrolled, so ptxas keeps it asynchronous without wg_tile_kloop's
// per-k-block commit and wait<1>, which the stem's shared-memory-bound walk cannot hide); 0: q.KH at run time, through wg_tile_kloop.
template <int N, int KS, class Epi, int KH_FIXED = 0>
__device__ __forceinline__ void row_strip(const CUtensorMap* mapWhi, const CUtensorMap* mapWlo, const RsParams& q) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    constexpr int LD = N + 4;
    constexpr uint32_t W_SBO = KS == 4 ? 1024u : 512u, W_LAYOUT = KS == 4 ? 2u : 4u;     // 128-byte (SWIZZLE_128B) or 64-byte (SWIZZLE_64B) weight rows
    const uint32_t slotb = 2u * (uint32_t)q.rowb;
    uint8_t* wsm = smem;                                                       // [KH][hi | lo] weight blocks
    uint8_t* ring = wsm + (((size_t)q.KH * 2 * q.w_block + 1023) & ~(size_t)1023);      // [RS_RING][hi | lo] image rows
    float* tile = reinterpret_cast<float*>(ring + (size_t)RS_RING * slotb);   // [128][LD] staged accumulator of one conv row
    uint8_t* extra = reinterpret_cast<uint8_t*>(tile + 128 * LD);             // [Epi::kExtraBytes]
    uint64_t* full = reinterpret_cast<uint64_t*>(extra + Epi::kExtraBytes);   // [RS_RING] producer -> consumers
    uint64_t* empty = full + RS_RING;            // [RS_RING] consumers (8 warps) -> producer
    uint64_t* fullW = empty + RS_RING;           // [1]

    const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
    const int units = q.B * q.nstrips * q.nseg;
    const int u0 = (int)blockIdx.x, ustep = (int)gridDim.x;

    if (threadIdx.x == 0) {
        for (int s = 0; s < RS_RING; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
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
                tma_load_2d(wsm + (size_t)ky * 2 * q.w_block, mapWhi, fullW, ky * KS * 16, 0);
                tma_load_2d(wsm + (size_t)ky * 2 * q.w_block + q.w_block, mapWlo, fullW, ky * KS * 16, 0);
            }
        }
        __syncwarp();
        int gl = 0;
        for (int u = u0; u < units; u += ustep) {
            const RsUnit U = Epi::unit(q, u);
            const int L = q.S * (U.T - 1) + q.KH;                   // image rows of the unit
            const int yi0 = q.S * U.y0 - q.P;
            const size_t xbyte = (size_t)q.xbyte0 + (size_t)U.strip * q.strip_bytes;
            for (int l = 0; l < L; ++l, ++gl) {
                const int slot = gl % RS_RING;
                mbar_wait(&empty[slot], ((gl / RS_RING) & 1) ^ 1);
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
                        const size_t off = ((size_t)U.b * q.H + yi) * (size_t)q.Wp * q.pxb + xbyte;
                        bulk_g2s(dst, q.in_hi + off, (uint32_t)q.rowb, &full[slot]);
                        bulk_g2s(dst + q.rowb, q.in_lo + off, (uint32_t)q.rowb, &full[slot]);
                    }
                }
                __syncwarp();
            }
        }
    } else {
        // ================= consumer warpgroups: MMAs of operand rows 64 wg .. 64 wg + 63, promotion, the kernel's epilogue =================
        const int wg = warp >> 2;
        int gl = 0;
        auto release = [&](int l) {                                    // local image row l of the unit
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[(gl + l) % RS_RING]);
        };
        auto keep = [](int) {};                                        // (ring rows are released per conv row, not per filter row)
        auto issued = [] {};
        mbar_wait(fullW, 0);
        const uint32_t wbase = smem_u32(wsm), rbase = smem_u32(ring) + (uint32_t)wg * 64u * 16u;
        Epi epi(q, extra, warp, lane);
        float tot[N / 2], c[N / 2];
        for (int u = u0; u < units; u += ustep) {
            const RsUnit U = Epi::unit(q, u);
            epi.begin(U);
            for (int t = 0; t < U.T; ++t) {
                // conv row t reads local image rows S t .. S t + KH - 1; rows up to S t + KH - S - 1 were waited for by earlier conv rows
                for (int l = (t == 0 ? 0 : q.S * t + q.KH - q.S); l < q.S * t + q.KH; ++l) mbar_wait(&full[(gl + l) % RS_RING], ((gl + l) / RS_RING) & 1);
#pragma unroll
                for (int k = 0; k < N / 2; ++k) tot[k] = 0.f;
                int ky = 0;                                            // k-block = filter row
                auto acquire = [&]() {
                    const uint32_t ra = rbase + (uint32_t)((gl + q.S * t + ky) % RS_RING) * slotb;
                    const uint32_t wa = wbase + (uint32_t)(ky * 2 * q.w_block);
                    ++ky;
                    return KbOperands{make_sdesc_ns(ra, 16u, 128u), make_sdesc_ns(ra + q.rowb, 16u, 128u), make_sdesc(wa, W_SBO, W_LAYOUT),
                                      make_sdesc(wa + q.w_block, W_SBO, W_LAYOUT), 0};
                };
                if constexpr (KH_FIXED > 0) {
                    auto walk = [&](auto mode) {
#pragma unroll
                        for (int ky0 = 0; ky0 < KH_FIXED; ky0 += RS_CHUNK) {
                            wg_fence();
#pragma unroll
                            for (int k = ky0; k < (ky0 + RS_CHUNK < KH_FIXED ? ky0 + RS_CHUNK : KH_FIXED); ++k) {
                                const KbOperands o = acquire();
                                wg_kblock<N, true, decltype(mode)::value, KS>(c, o.dA, o.dAlo, o.dB, o.dBlo, k == ky0);
                            }
                            wg_commit();
                            wg_wait<0>();
                            wg_promote(tot, c);
                        }
                    };
                    if (q.dbg & 1) walk(tc_int<1>()); else walk(tc_int<0>());
                } else {
                    if (q.dbg & 1) wg_tile_kloop<N, true, 1, KS>(tot, c, q.KH, RS_CHUNK, acquire, keep, issued);
                    else wg_tile_kloop<N, true, 0, KS>(tot, c, q.KH, RS_CHUNK, acquire, keep, issued);
                }
                for (int l = q.S * t; l < q.S * (t + 1); ++l) release(l);      // not read by the next conv row
                consumers_sync();                                      // the previous conv row's staged accumulator has been read
                wg_stage<N>(tot, tile, LD, wg, warp, lane);
                consumers_sync();
                epi.row(U, t, tile);
            }
            const int L = q.S * (U.T - 1) + q.KH;
            for (int l = q.S * U.T; l < L; ++l) release(l);
            gl += L;
        }
        epi.finish();
    }
}

// row_conv_kernel: conv row y0 + t of the unit -> bias [+ ReLU] -> fp32 and / or planes.  Thread = operand row r (output column r / RS when
// r % RS == 0), channels [half N / 2, +N / 2).
template <int N>
struct RowConvEpi {
    static constexpr int kExtraBytes = 0;
    static __device__ __forceinline__ RsUnit unit(const RsParams& q, int u) {
        RsUnit U;
        rs_segment(q, u, q.Ho, U.b, U.strip, U.y0, U.T);
        return U;
    }
    const RsParams& q;
    const int r, half;
    int x;
    bool ok;
    float amax = 0.f;
    __device__ __forceinline__ RowConvEpi(const RsParams& q_, uint8_t*, int warp, int lane) : q(q_), r((warp & 3) * 32 + lane), half(warp >> 2) {}
    __device__ __forceinline__ void begin(const RsUnit& U) {
        x = U.strip * q.pxs + r / q.RS;
        ok = (r % q.RS) == 0 && x < q.Wo && !(q.dbg & 16);
    }
    __device__ __forceinline__ void row(const RsUnit& U, int t, const float* tile) {
        if (!ok) return;
        const float osc = q.out_scale;
        const float* acc = tile + r * (N + 4);
        const long long pix = ((long long)U.b * q.Ho + (U.y0 + t)) * q.out_W + q.out_xoff + x;
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
    __device__ __forceinline__ void finish() { if (q.out_hi) note_fp16_range(amax, q.range_flag); }
};

template <int N, int KS>
__global__ void __launch_bounds__(RS_THREADS, 1)
row_conv_kernel(const __grid_constant__ CUtensorMap mapWhi, const __grid_constant__ CUtensorMap mapWlo, const __grid_constant__ RsParams q) {
    row_strip<N, KS, RowConvEpi<N>>(&mapWhi, &mapWlo, q);
}

constexpr int SP_KH = 7, SP_STRIDE = 2, SP_PAD = 3;
constexpr int SP_XOFF = 5;                       // zero pixels in front of every row of the planes (pad 3 + 2: column -1 of strip 0 stays in the row)
constexpr int SP_CENTERS = 63;                   // pooled columns per strip (conv columns 126 t - 1 .. 126 t + 126)

// stem_pool_kernel: thread = conv column x of the strip (conv column 126 strip - 1 + x), channels [32 half, +32).  Conv row 2 i - 1 opens
// pooled row i, conv row 2 i + 1 closes it (and opens pooled row i + 1).
struct StemPoolEpi {
    static constexpr int kExtraBytes = 2 * 2 * 4 * 32 * sizeof(float);     // [2 parities][2 halves][4 quadrants][32]: column maxima of each warp's column 0
    static __device__ __forceinline__ RsUnit unit(const RsParams& q, int u) {
        RsUnit U;
        int i0, nrows;
        rs_segment(q, u, q.Hq, U.b, U.strip, i0, nrows);       // pooled rows i0 .. i0 + nrows - 1 (>= 1 by construction of nseg)
        U.y0 = 2 * i0 - 1; U.T = 2 * nrows + 1;
        return U;
    }
    const RsParams& q;
    float* edge;
    const int lane, qd, half, x, cb;
    int j, ntile = 0;
    bool col_ok, centre;
    float amax = 0.f;
    // run[k] = column-wise maximum of the conv rows of the pooled row that is open (vertical max first: the horizontal 3-max, its shuffles and
    // the cross-warp exchange are then needed only once per pooled row, on the maximum of the three conv rows)
    float run[32];
    __device__ __forceinline__ StemPoolEpi(const RsParams& q_, uint8_t* extra, int warp, int lane_)
        : q(q_), edge(reinterpret_cast<float*>(extra)), lane(lane_), qd(warp & 3), half(warp >> 2), x((warp & 3) * 32 + lane_), cb((warp >> 2) * 32) {}
    __device__ __forceinline__ void begin(const RsUnit& U) {
        const int cc0 = 126 * U.strip - 1 + x;                         // conv column
        col_ok = cc0 >= 0 && cc0 < q.Wo;
        const int jl = (x - 1) >> 1;                                   // pooled column inside the strip (x odd)
        j = SP_CENTERS * U.strip + jl;
        centre = (x & 1) && jl < SP_CENTERS && j < q.Wq;
    }
    __device__ __forceinline__ void row(const RsUnit& U, int t, const float* stage) {
        const float osc = q.out_scale;
        float acc[32];
        {
            const float* sp = stage + x * (64 + 4) + cb;
#pragma unroll
            for (int k = 0; k < 32; k += 4) {
                const float4 v = *reinterpret_cast<const float4*>(sp + k);
                acc[k] = v.x; acc[k + 1] = v.y; acc[k + 2] = v.z; acc[k + 3] = v.w;
            }
        }
        const int y = U.y0 + t;                                        // conv row
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
            // conv row 2i + 1 closes pooled row i: column maxima of its three conv rows, then the horizontal 3-max
            const int i = ((U.y0 + 1) >> 1) + (t >> 1) - 1;
#pragma unroll
            for (int k = 0; k < 32; ++k) run[k] = fmaxf(run[k], acc[k]);
            float* ed = edge + (((ntile & 1) * 2 + half) * 4) * 32;
            ++ntile;
            if (lane == 0) {                                           // column 32 (qd + 1) of the strip is lane 31's right neighbour
#pragma unroll
                for (int k = 0; k < 32; k += 4) *reinterpret_cast<float4*>(ed + qd * 32 + k) = make_float4(run[k], run[k + 1], run[k + 2], run[k + 3]);
            }
            asm volatile("bar.sync 1, 256;" ::: "memory");
            const bool last_lane = lane == 31;
            const float* en = ed + ((qd + 1) & 3) * 32;
            const bool wrap = qd == 3;                                 // column 128 does not exist (and column 127 is no centre)
            const long long pix = ((long long)U.b * q.Hq + i) * q.Wq + j;
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
            for (int k = 0; k < 32; ++k) run[k] = acc[k];              // conv row 2i + 1 is also the first row of pooled row i + 1
        }
    }
    __device__ __forceinline__ void finish() { if (q.out_hi) note_fp16_range(amax, q.range_flag); }
};

__global__ void __launch_bounds__(RS_THREADS, 1)
stem_pool_kernel(const __grid_constant__ CUtensorMap mapWhi, const __grid_constant__ CUtensorMap mapWlo, const __grid_constant__ RsParams q) {
    row_strip<64, 2, StemPoolEpi, SP_KH>(&mapWhi, &mapWlo, q);
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

// ---- host ----

// staged bytes per image row and plane: operand rows 0..127 at a 16-byte pitch, KS * 32 bytes each
static int rs_rowb(int KS) { return (127 * 16 + KS * 32 + 15) / 16 * 16; }

// the conv geometry both kernels share: KH filter rows of KS K steps into N channels, stride S, padding P, planes of pxb bytes per pixel
static void rs_conv(RsParams& q, int KH, int S, int P, int KS, int pxb, int N) {
    q.KH = KH; q.S = S; q.P = P; q.KS = KS; q.pxb = pxb; q.RS = S * pxb / 16;
    q.rowb = rs_rowb(KS);
    q.w_block = N * KS * 32;
    { const char* e = getenv("VD3D_TC_DEBUG"); q.dbg = e ? atoi(e) : 0; }
}

// Row segments per strip: the split of `rows` (conv or pooled) into at most nmax segments that minimises the rounds of `slots` CTAs times the
// conv rows a unit computes (a * rows per segment + c).
static void rs_partition(RsParams& q, int rows, int nmax, int slots, int a, int c) {
    long long best = -1;
    for (int n = 1; n <= nmax && n <= rows; ++n) {
        const int seg_rows = (rows + n - 1) / n;
        const int nseg = (rows + seg_rows - 1) / seg_rows;
        const long long units = (long long)q.B * q.nstrips * nseg;
        const long long cost = ((units + slots - 1) / slots) * ((long long)a * seg_rows + c);
        if (best < 0 || cost < best) { best = cost; q.nseg = nseg; q.seg_rows = seg_rows; }
    }
}

static size_t rs_smem(const RsParams& q, int N, int extra) {
    return (((size_t)q.KH * 2 * q.w_block + 1023) & ~(size_t)1023) + (size_t)RS_RING * 2 * q.rowb + (size_t)128 * (N + 4) * sizeof(float) + extra +
           (2 * RS_RING + 1) * sizeof(uint64_t) + 1024;
}

// weights = [N][KH * KS * 16] fp16 (hi, lo) matrices (k = ky * KS * 16 + kx * pc + c)
template <auto Kernel>
static int rs_launch(const RsParams& q, int N, const void* w_hi, const void* w_lo, int grid, size_t smem, void* stream, const char* what) {
    CUtensorMap mWhi, mWlo;
    int rc;
    if ((rc = make_map_wgt(&mWhi, w_hi, N, q.KH * q.KS * 16, N, 2, q.KS * 32))) return rc;
    if ((rc = make_map_wgt(&mWlo, w_lo, N, q.KH * q.KS * 16, N, 2, q.KS * 32))) return rc;
    const cudaError_t le = tc_launch<Kernel>(grid, RS_THREADS, smem, stream, mWhi, mWlo, q);
    if (le != cudaSuccess) { set_error("%s: launch failed: %s", what, cudaGetErrorString(le)); return VD3D_ECUDA; }
    VD3D_CHECK_LAUNCH(what);
    return VD3D_OK;
}

}  // namespace vd3d

using namespace vd3d;

static int image_to_h16_rows(const float* img, int B, int C, int H, int W, void* hi16, void* lo16, int Wp, int xoff, int cpad, void* stream, const char* what) {
    const long long total = (long long)B * H * W;
    image_to_h16_rows_c_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(img, (__half*)hi16, (__half*)lo16, C, H, W, total, Wp, xoff, cpad, fp16_range_flag());
    VD3D_CHECK_LAUNCH(what);
    return VD3D_OK;
}

extern "C" int vd3d_image_to_h16_rows(const float* img, int B, int C, int H, int W, void* hi16, void* lo16, int Wp, int xoff, void* stream) {
    VD3D_REQUIRE(img && hi16 && lo16 && B > 0 && C >= 1 && C <= 4 && H > 0 && W > 0 && xoff >= 0 && Wp >= W + xoff, "image_to_h16_rows: bad args");
    return image_to_h16_rows(img, B, C, H, W, hi16, lo16, Wp, xoff, 4, stream, "image_to_h16_rows");
}

extern "C" int vd3d_image_to_h16_rows_c(const float* img, int B, int C, int H, int W, void* hi16, void* lo16, int Wp, int xoff, int cpad, void* stream) {
    VD3D_REQUIRE(img && hi16 && lo16 && B > 0 && C >= 1 && (cpad == 4 || cpad == 8) && C <= cpad && H > 0 && W > 0 && xoff >= 0 && Wp >= W + xoff, "image_to_h16_rows_c: bad args");
    return image_to_h16_rows(img, B, C, H, W, hi16, lo16, Wp, xoff, cpad, stream, "image_to_h16_rows_c");
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
    const long long bytes = (long long)(xoff - P) * pxb + 2048LL * (nstrips - 1) + rs_rowb(KS);
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
    RsParams q;
    memset(&q, 0, sizeof(q));
    q.in_hi = (const uint8_t*)in_hi; q.in_lo = (const uint8_t*)in_lo; q.B = B; q.H = H; q.Wp = Wp;
    rs_conv(q, KH, S, P, KW * pc * 2 <= 64 ? 2 : 4, pc * 2, N);
    VD3D_REQUIRE(KH >= S, "row_conv: KH >= stride");
    VD3D_REQUIRE(((xoff - P) * q.pxb) % 16 == 0, "row_conv: (xoff - pad) pixels must be a multiple of 16 bytes");
    q.xbyte0 = (xoff - P) * q.pxb; q.strip_bytes = 2048;
    q.Ho = (H + 2 * P - KH) / S + 1; q.Wo = (W + 2 * P - KW) / S + 1;
    VD3D_REQUIRE(q.Ho > 0 && q.Wo > 0, "row_conv: empty output");
    VD3D_REQUIRE(out_W >= q.Wo + out_xoff, "row_conv: output row pitch too small");
    q.pxs = 128 / q.RS; q.nstrips = (q.Wo + q.pxs - 1) / q.pxs;
    rs_partition(q, q.Ho, 32, 2 * kNumSMs, 1, KH);
    q.out_scale = out_scale; q.bias = bias; q.relu = relu;
    q.out = out; q.out_hi = (__half*)out_hi16; q.out_lo = (__half*)out_lo16; q.out_W = out_W; q.out_xoff = out_xoff; q.out_cs = out_cs; q.out_co = out_co;
    q.range_flag = out_hi16 ? fp16_range_flag() : nullptr;
    const size_t smem = rs_smem(q, N, 0);
    VD3D_REQUIRE(smem <= 227 * 1024, "row_conv: shared-memory budget exceeded");
    const int units = B * q.nstrips * q.nseg;
    const int slots = smem <= 110 * 1024 ? 2 * kNumSMs : kNumSMs;        // two CTAs per SM when they fit: one hides the other's per-row hand-offs
    const int grid = units < slots ? units : slots;
    if (N == 16) return q.KS == 2 ? rs_launch<row_conv_kernel<16, 2>>(q, N, w_hi, w_lo, grid, smem, stream, "row_conv")
                                  : rs_launch<row_conv_kernel<16, 4>>(q, N, w_hi, w_lo, grid, smem, stream, "row_conv");
    return q.KS == 2 ? rs_launch<row_conv_kernel<32, 2>>(q, N, w_hi, w_lo, grid, smem, stream, "row_conv")
                     : rs_launch<row_conv_kernel<32, 4>>(q, N, w_hi, w_lo, grid, smem, stream, "row_conv");
}

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
    RsParams q;
    memset(&q, 0, sizeof(q));
    q.in_hi = (const uint8_t*)in_hi; q.in_lo = (const uint8_t*)in_lo; q.B = B; q.H = H; q.Wp = Wp;
    rs_conv(q, SP_KH, SP_STRIDE, SP_PAD, 2, 8, 64);
    q.xbyte0 = 0; q.strip_bytes = 126 * 16;                           // strip t starts at conv column 126 t - 1, i.e. padded pixel 252 t
    q.Ho = (H + 2 * SP_PAD - SP_KH) / SP_STRIDE + 1; q.Wo = (W + 2 * SP_PAD - SP_KH) / SP_STRIDE + 1;
    VD3D_REQUIRE(q.Ho > 0 && q.Wo > 0, "stem_pool_fused: empty output");
    q.Hq = (q.Ho + 2 - 3) / 2 + 1; q.Wq = (q.Wo + 2 - 3) / 2 + 1;
    q.nstrips = (q.Wq + SP_CENTERS - 1) / SP_CENTERS;
    rs_partition(q, q.Hq, 16, kNumSMs, 2, 1);                          // every unit recomputes one conv row of its upper neighbour
    q.out_scale = out_scale; q.bias = bias; q.out = out; q.out_hi = (__half*)out_hi16; q.out_lo = (__half*)out_lo16; q.out_cs = out_cs; q.out_co = out_co;
    q.range_flag = out_hi16 ? fp16_range_flag() : nullptr;
    const int units = B * q.nstrips * q.nseg;
    return rs_launch<stem_pool_kernel>(q, 64, w_hi, w_lo, units < kNumSMs ? units : kNumSMs, rs_smem(q, 64, StemPoolEpi::kExtraBytes), stream, "stem_pool_fused");
}
