// Pieces of the wgmma conv engine shared by conv2d_tc.cu (dense convolutions) and dcn_fused.cu (deformable convolutions whose
// A operand is gathered into shared memory by the kernel itself): kernel parameters, the k-block MMA sequence, the persistent kernels'
// epilogue (staged accumulator -> scale / bias / residual / ReLU -> fp32 value and / or fp16 (hi, lo) planes), the tile order, and host helpers.
#pragma once
#include "tc_common.cuh"
#include <cstdlib>
#include <type_traits>

namespace vd3d {

constexpr int TC_TW = 16, TC_TH = 8;          // output tile = 8 rows x 16 columns = 128 pixels (two 64-row warpgroup MMAs)
constexpr int TC_MAX_BN = 128;                // widest tile: the chunk accumulator and its promoted sum take BN registers per consumer thread
// Warp roles of the tensor-core kernels: warps 0..7 = two consumer warpgroups (warpgroup w issues the MMAs of tile rows 64 w .. 64 w + 63,
// promotes the chunks and runs the epilogue), the warps after them produce the operands.
constexpr int TC_CONSUMERS = 256;

constexpr int TC_MAX_LEVELS = 5;
struct TcLevel {
    int Ho, Wo, tiles_w, tiles_h, m_begin, res_H, res_W;
    int pad_h, pad_w;        // tap origin: input row / column of tap (0, 0) for output (0, 0) is (-pad_h, -pad_w)
    int w_row;               // first weight row of the level (the levels of a transposed conv each own Cout rows of one matrix)
    int up;                  // 1: output pixel (ho, wo) of image b is pixel (2 ho, 2 wo) of a [B][2 Ho][2 Wo] tensor, plus pix_off (sub-pixel phase)
    long long pix_off, res_off;
};

struct TcParams {
    int B, H, W, Cin, KH, KW, pad, dil, stride;
    int Ho, Wo, Cout, BN, stages, passes, chunk;
    int f16;                 // 0: tf32 operands (32 channels / k-block), 1: fp16 hi/lo operands (64 channels / k-block)
    int bk;                  // channels per k-block
    int cin_pad;             // weight K layout: per-tap channel count rounded up to bk
    float out_scale;         // multiplies the accumulator (undoes the power-of-two weight scaling of the fp16 path)
    void* out_h16_hi; void* out_h16_lo;
    int* range_flag;         // fp16-range guard (common.cuh): ORed to 1 when a value written to the fp16 planes is beyond the fp16 range
    int tiles_w, tiles_h;
    int stride_w, pad_w;     // W-direction stride / padding (the H direction uses stride / pad); equal to them for ordinary convs
    int m_tiles, n_tiles;    // persistent kernel: tile counts along M (B * tiles_h * tiles_w) and N
    // fused 3x3 / stride-2 / pad-1 max-pool of the (ReLU) output (the ResNet stem, resnet.py:186-189): when pool_out != nullptr the epilogue
    // does not write the conv output at all; it pools every tile in shared memory and writes the pooled tensor
    float* pool_out; int pool_cs, pool_co, pool_H, pool_W;
    int two_pass;            // error-budget experiments (vd3d_conv2d_tc16 passes = 2): drop the A_lo * W_hi product (activations then carry 11 significant bits)
    int mblock;              // persistent kernels: scheduling units (tiles) per M block of the L2-aware tile order (0: one block)
    int rowb;                // bytes per operand row in shared memory = K bytes per k-block: 128 (SWIZZLE_128B) or 64 (32 fp16, SWIZZLE_64B)
    // conv2d_tcp_kernel: where the accumulator is staged for the epilogue.  1: in the operand stage of the tile's last k-block, held until the
    // epilogue is done (no separate staging tile: one more stage fits); 0: a separate tile after the ring
    int tile_in_ring;
    int split_stage;         // (tile_in_ring, epilogue warps) rows 64..127 of the staged accumulator go to a half tile after the ring
    int cout_pad;           // Cout rounded up to 16 (ragged last N tile = cout_pad - (n_tiles - 1) * BN columns)
    int v8;                  // output / residual / bias slices are 32-byte aligned (fp16 plane slices then take 16-byte accesses)
    long long* trace; int trace_n;   // VD3D diagnostics (vd3d_tc_set_trace): clock64 stamps of CTA 0, [12][trace_n]: rows 0..4 and 9 per k-block, 5..8, 10 and 11 per tile
    int dbg;                 // timing experiments only (VD3D_TC_DEBUG; results are wrong): bit 0 = one MMA per k-step, bit 1 = skip the lo-plane loads, bit 4 = no epilogue output, bit 5 = no residual loads
    int out_cs, out_co, res_cs, res_co, relu;
    const float* bias; const float* res; float* out; float* out_lo;
    const void* res_h16_hi; const void* res_h16_lo;   // residual given as fp16 (hi, lo) planes (value = hi + lo) instead of an fp32 tensor (`res`)
    int res_up_H, res_up_W;  // > 0: the residual is [B][res_up_H][res_up_W] at half the output resolution, read nearest-upsampled (tcp_res_pix)
    // Multi-level launch (vd3d_conv2d_tc16 with L > 1; n_levels = 0: one tensor).  The M tiles of the levels are concatenated: level l owns tiles
    // [m_begin, m_begin + B * tiles_h * tiles_w) and reads its own activation maps; its output (residual) pixel p sits at pixel pix_off + p
    // (res_off + p, or of the [B][res_H][res_W] half-resolution residual when res_W > 0) of the `out` (`res`) pointers.
    // vd3d_convtranspose2d_tc16 runs the four sub-pixel phases of a 4x4 / stride-2 transposed conv as four levels over ONE input: each with
    // its own tap origin, weight rows and interleaved output pixels (TcLevel::pad_h / pad_w / w_row / up).
    int n_levels;
    TcLevel lv[TC_MAX_LEVELS];
    // Tile-listed launch (vd3d_conv2d_tc16_tiles; one level, stride 1): the M tiles are the entries (b, y0, x0, 0) of `tlist`, 8 x 16 output tiles
    // whose origin may be any pixel, and there are tcount[0] of them (read on the device, so the list can be built by an earlier kernel of the
    // stream); only the pixels whose byte of `smap` [B][Ho][Wo] is set are stored (and feed the fp16-range guard).  m_tiles stays the dense
    // count: it sizes the grid and the L2 blocks.
    const int4* tlist; const int* tcount; const uint8_t* smap;
};

// 8 consecutive channels (16-byte aligned)
__device__ __forceinline__ void ld8(const float* ptr, float (&v)[8]) {
    const float4 a = ldg4(ptr), b = ldg4(ptr + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
// 8 consecutive channels of a tensor kept as fp16 (hi, lo) planes: value = hi + lo (exact in fp32: |lo| <= ulp16(hi) / 2)
__device__ __forceinline__ void ld8_planes(const __half* hp, const __half* lp, bool v8, float (&v)[8]) {
    uint32_t h[4], l[4];
    if (v8) {
        const uint4 a = __ldg(reinterpret_cast<const uint4*>(hp)), b = __ldg(reinterpret_cast<const uint4*>(lp));
        h[0] = a.x; h[1] = a.y; h[2] = a.z; h[3] = a.w; l[0] = b.x; l[1] = b.y; l[2] = b.z; l[3] = b.w;
    } else {
        const uint2 a0 = __ldg(reinterpret_cast<const uint2*>(hp)), a1 = __ldg(reinterpret_cast<const uint2*>(hp + 4));
        const uint2 b0 = __ldg(reinterpret_cast<const uint2*>(lp)), b1 = __ldg(reinterpret_cast<const uint2*>(lp + 4));
        h[0] = a0.x; h[1] = a0.y; h[2] = a1.x; h[3] = a1.y; l[0] = b0.x; l[1] = b0.y; l[2] = b1.x; l[3] = b1.y;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 fh = __half22float2(*reinterpret_cast<const __half2*>(&h[i])), fl = __half22float2(*reinterpret_cast<const __half2*>(&l[i]));
        v[2 * i] = fh.x + fl.x; v[2 * i + 1] = fh.y + fl.y;
    }
}
__device__ __forceinline__ void ld4_planes(const __half* hp, const __half* lp, float (&v)[8]) {
    const uint2 a = __ldg(reinterpret_cast<const uint2*>(hp)), b = __ldg(reinterpret_cast<const uint2*>(lp));
    const uint32_t h[2] = {a.x, a.y}, l[2] = {b.x, b.y};
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const float2 fh = __half22float2(*reinterpret_cast<const __half2*>(&h[i])), fl = __half22float2(*reinterpret_cast<const __half2*>(&l[i]));
        v[2 * i] = fh.x + fl.x; v[2 * i + 1] = fh.y + fl.y;
    }
}
__device__ __forceinline__ void st8(float* ptr, const float (&v)[8]) {
    *reinterpret_cast<float4*>(ptr) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>(ptr + 4) = make_float4(v[4], v[5], v[6], v[7]);
}
__device__ __forceinline__ uint32_t pack_h2(__half a, __half b) { __half2 h = __halves2half2(a, b); return *reinterpret_cast<uint32_t*>(&h); }
// fp16 (hi, lo) planes of 4 values: hi = rn16(v), lo = rn16(v - hi)
__device__ __forceinline__ void split4(const float* v, uint2& hv, uint2& lv) {
    __half h0 = __float2half_rn(v[0]), h1 = __float2half_rn(v[1]), h2 = __float2half_rn(v[2]), h3 = __float2half_rn(v[3]);
    hv.x = pack_h2(h0, h1); hv.y = pack_h2(h2, h3);
    lv.x = pack_h2(__float2half_rn(v[0] - __half2float(h0)), __float2half_rn(v[1] - __half2float(h1)));
    lv.y = pack_h2(__float2half_rn(v[2] - __half2float(h2)), __float2half_rn(v[3] - __half2float(h3)));
}

// Tile order of the persistent kernels.  Unit u -> (mu, nt): M fastest inside an M BLOCK of `mblock` units, then the N tiles, then the
// next M block.  With one block (mblock == 0) every N tile streams the whole activation tensor again; with blocks sized to stay
// L2-resident the activations are read from DRAM once and the weights once per block.  Pure scheduling: every tile computes the same bits.
__device__ __forceinline__ void unit_tile(const TcParams& p, int u, int mt_units, int& mu, int& nt) {
    if (p.mblock <= 0 || p.mblock >= mt_units) { mu = u % mt_units; nt = u / mt_units; return; }
    const int per = p.mblock * p.n_tiles;
    const int blk = u / per, r = u - blk * per;
    const int m0 = blk * p.mblock;
    const int cur = min(p.mblock, mt_units - m0);
    nt = r / cur; mu = m0 + (r - nt * cur);
}
__device__ __forceinline__ int unit_nt(const TcParams& p, int u, int mt_units) { int mu, nt; unit_tile(p, u, mt_units, mu, nt); return nt; }

// One k-block of MMAs of a consumer warpgroup: KSTEPS K steps of 32 bytes (16 fp16 / 8 tf32) inside the operand rows, three products per
// step (A_lo W_hi, A_hi W_lo, A_hi W_hi: small terms first, then the main product), one (A W) or two (A W_lo, A W) in the experiment modes.
// `first`: the first k-block of a promotion chunk (the accumulator restarts from zero).  MODE and KSTEPS are template arguments so that the
// MMA chain is straight-line code: wgmma instructions under a run-time branch make ptxas serialise them (warpgroup.arrive / wait injection).
// AK: step of the A descriptor per K step in 16-byte units (2: 32 bytes along a swizzled 128-byte row; conv2d_row64.cu's core-matrix rows
// keep each 8-channel group in a plane of its own, so a K step there moves two planes).
template <int N, bool F16>
__device__ __forceinline__ void wg_mma(float (&c)[N / 2], uint64_t da, uint64_t db, uint32_t acc) {
    if constexpr (F16) wgmma_f16<N>(c, da, db, acc); else wgmma_tf32<N>(c, da, db, acc);
}
template <int N, bool F16, int MODE, int KSTEPS, int AK = 2>
__device__ __forceinline__ void wg_kblock(float (&c)[N / 2], uint64_t dA, uint64_t dAlo, uint64_t dB, uint64_t dBlo, bool first) {
#pragma unroll
    for (int k = 0; k < KSTEPS; ++k) {
        const uint64_t off = (uint64_t)((k * 32) >> 4), aoff = (uint64_t)(k * AK);
        const uint32_t acc0 = (first && k == 0) ? 0u : 1u;
        if constexpr (MODE == 0) {
            wg_mma<N, F16>(c, dAlo + aoff, dB + off, acc0);
            wg_mma<N, F16>(c, dA + aoff, dBlo + off, 1u);
            wg_mma<N, F16>(c, dA + aoff, dB + off, 1u);
        } else if constexpr (MODE == 2) {
            wg_mma<N, F16>(c, dA + aoff, dBlo + off, acc0);
            wg_mma<N, F16>(c, dA + aoff, dB + off, 1u);
        } else {
            wg_mma<N, F16>(c, dA + aoff, dB + off, acc0);
        }
    }
}
// MMA mode of a TcParams launch: 0 = three products (production), 1 = one (passes == 1 or the VD3D_TC_DEBUG bit 0 experiment), 2 = two
__host__ __device__ __forceinline__ int tc_mma_mode(const TcParams& p) { return (p.passes == 1 || (p.dbg & 1)) ? 1 : (p.two_pass ? 2 : 0); }

// Chunked promotion: the tensor core adds every product into the fp32 accumulator with truncation, so the K loop is cut into chunks of
// `chunk` k-blocks, each accumulated from zero in a chunk accumulator and then added with round-to-nearest into the per-thread sum `tot`.
template <int R> __device__ __forceinline__ void wg_promote(float (&tot)[R], float (&c)[R]) {
    wg_fence_regs(c);
#pragma unroll
    for (int i = 0; i < R; ++i) tot[i] += c[i];
}

// Shared-memory operands of one k-block, and the ring slot to hand back to the producers once its MMAs have completed.
struct KbOperands { uint64_t dA, dAlo, dB, dBlo; int slot; };

// One k-block: wait for its operands (acquire), issue its MMAs as one commit group, then wait until at most this group is outstanding and
// release the slot of the previous k-block.  `pend`: slot of the k-block whose MMAs may still be running (-1: none).
template <int N, bool F16, int MODE, int KSTEPS, int AK = 2, class Acquire, class Release, class Issued>
__device__ __forceinline__ void wg_kblock_step(float (&c)[N / 2], bool first, int& pend, Acquire& acquire, Release& release, Issued& issued) {
    const KbOperands o = acquire();
    wg_fence();
    wg_kblock<N, F16, MODE, KSTEPS, AK>(c, o.dA, o.dAlo, o.dB, o.dBlo, first);
    wg_commit();
    wg_wait<1>();                                       // every earlier k-block's MMAs are done
    if (pend >= 0) release(pend);
    pend = o.slot;
    issued();
}
// K loop of one tile of a consumer warpgroup: KB k-blocks in chunks of `chunk`, the sum of the chunks in `tot` (which the caller zeroes).
// Inside a chunk one k-block of MMAs stays in flight while the next one is issued; the chunk ends with a drain (wait 0) and its promotion.
// The loop over a chunk's k-blocks is an inner loop and the promotion sits after it, never under a branch inside it: then no instruction
// other than a wgmma touches the accumulator on a path where a wgmma writing it may still be outstanding, and ptxas keeps the chain
// asynchronous (with a conditional promotion inside the k-block loop it injects a warpgroup.wait that drains the pipe after every k-block).
// `keep_last`: the slot of the tile's last k-block is not released but returned (the caller stages the accumulator there and releases it after
// the epilogue); otherwise every slot is released and the result is -1.
template <int N, bool F16, int MODE, int KSTEPS, int AK = 2, class Acquire, class Release, class Issued>
__device__ __forceinline__ int wg_tile_kloop(float (&tot)[N / 2], float (&c)[N / 2], int KB, int chunk, Acquire& acquire, Release& release, Issued& issued,
                                             bool keep_last = false) {
    int pend = -1;
    for (int kb0 = 0; kb0 < KB; kb0 += chunk) {
        const int kb1 = min(KB, kb0 + chunk);
        pend = -1;
        wg_kblock_step<N, F16, MODE, KSTEPS, AK>(c, true, pend, acquire, release, issued);
        for (int kb = kb0 + 1; kb < kb1; ++kb) wg_kblock_step<N, F16, MODE, KSTEPS, AK>(c, false, pend, acquire, release, issued);
        wg_wait<0>();
        if (!keep_last || kb1 < KB) { release(pend); pend = -1; }
        wg_promote(tot, c);
    }
    return pend;
}
template <int V> using tc_int = std::integral_constant<int, V>;

// Epilogue arithmetic of the persistent kernels, per 8 output channels n .. n + 7 of one output pixel `pix` (n + 4 <= Cout; when n + 8 > Cout,
// the Cout % 8 == 4 tail, only the first four are read and written).  Split in two so that an epilogue can have the residual loads of
// several groups in flight before it computes the first.
// Output geometry of M tile mu: the output pixel of the tile's (0, 0) (a multiple of the tile size, or a list entry's origin), image, the output size, and the pixel offsets of the output and the residual (the level's,
// in a multi-level launch; zero otherwise).  The level table is indexed with compile-time indices only, so it stays in parameter space.
// Tap origin (pad_h, pad_w), first weight row (w_row) and output pixel map (up) of the tile's level: p.pad / p.pad_w, 0 and 0 outside
// multi-level launches.
struct TcGeom { int w0, h0, b, Ho, Wo, lvl, res_H, res_W, pad_h, pad_w, w_row, up; long long pix_off, res_off; };
__device__ __forceinline__ TcGeom tile_geom(const TcParams& p, int mu) {
    TcGeom g;
    g.lvl = 0; g.Ho = p.Ho; g.Wo = p.Wo; g.res_H = p.res_up_H; g.res_W = p.res_up_W; g.pix_off = 0; g.res_off = 0;
    g.pad_h = p.pad; g.pad_w = p.pad_w; g.w_row = 0; g.up = 0;
    if (p.tlist) {
        const int4 e = __ldg(p.tlist + mu);
        g.b = e.x; g.h0 = e.y; g.w0 = e.z;
        return g;
    }
    int tiles_w = p.tiles_w, tiles_h = p.tiles_h;
    if (p.n_levels > 0) {
#pragma unroll
        for (int i = 0; i < TC_MAX_LEVELS; ++i)
            if (i < p.n_levels && mu >= p.lv[i].m_begin) {
                g.lvl = i; g.Ho = p.lv[i].Ho; g.Wo = p.lv[i].Wo; g.res_H = p.lv[i].res_H; g.res_W = p.lv[i].res_W;
                g.pix_off = p.lv[i].pix_off; g.res_off = p.lv[i].res_off; tiles_w = p.lv[i].tiles_w; tiles_h = p.lv[i].tiles_h;
                g.pad_h = p.lv[i].pad_h; g.pad_w = p.lv[i].pad_w; g.w_row = p.lv[i].w_row; g.up = p.lv[i].up;
            }
#pragma unroll
        for (int i = 0; i < TC_MAX_LEVELS; ++i)
            if (i == g.lvl) mu -= p.lv[i].m_begin;
    }
    g.w0 = (mu % tiles_w) * TC_TW; mu /= tiles_w;
    g.h0 = (mu % tiles_h) * TC_TH; g.b = mu / tiles_h;
    return g;
}
// Whether the epilogue stores output pixel (ho, wo) of the tile: inside the output and (tile-listed launches) set in the store map.
__device__ __forceinline__ bool tcp_stores(const TcParams& p, const TcGeom& g, int ho, int wo) {
    return ho < g.Ho && wo < g.Wo && (!p.smap || __ldg(p.smap + ((long long)g.b * g.Ho + ho) * g.Wo + wo));
}
// M tiles of a launch: the dense count, or the device count of a tile-listed launch (read after pdl_wait)
__device__ __forceinline__ int tcp_m_tiles(const TcParams& p) { return p.tcount ? __ldg(p.tcount) : p.m_tiles; }
// Output pixel of (b, ho, wo), and its residual pixel: the same pixel, or (res_W > 0) pixel (ho >> 1, wo >> 1) of the half-resolution
// residual, i.e. the nearest-neighbour x2 upsampling of the FPN top-down path fused into the residual read.  A sub-pixel phase level (up = 1)
// writes pixel (2 ho, 2 wo) of the [B][2 Ho][2 Wo] output; its pix_off (2 W r + s for phase (r, s)) picks the phase's pixel of each 2x2 cell.
__device__ __forceinline__ long long tcp_out_pix(const TcGeom& g, int ho, int wo) {
    return g.pix_off + ((((long long)g.b * g.Ho + ho) * g.Wo) << (2 * g.up)) + ((long long)wo << g.up);
}
__device__ __forceinline__ long long tcp_res_pix(const TcGeom& g, int ho, int wo) {
    return g.res_off + (g.res_W > 0 ? ((long long)g.b * g.res_H + (ho >> 1)) * g.res_W + (wo >> 1) : ((long long)g.b * g.Ho + ho) * g.Wo + wo);
}
// (1) the residual (zeros without one)
__device__ __forceinline__ void tcp_epi_res(const TcParams& p, long long pix, int n, float (&rr)[8]) {
#pragma unroll
    for (int k = 0; k < 8; ++k) rr[k] = 0.f;
    if (p.dbg & 32) return;
    const bool full8 = n + 8 <= p.Cout;
    if (p.res) {
        const float* rp = p.res + pix * p.res_cs + p.res_co + n;
        if (full8) ld8(rp, rr);
        else { const float4 t4 = ldg4(rp); rr[0] = t4.x; rr[1] = t4.y; rr[2] = t4.z; rr[3] = t4.w; }
    } else if (p.res_h16_hi) {
        const __half* rph = reinterpret_cast<const __half*>(p.res_h16_hi) + pix * p.res_cs + p.res_co + n;
        const __half* rpl = reinterpret_cast<const __half*>(p.res_h16_lo) + pix * p.res_cs + p.res_co + n;
        if (full8) ld8_planes(rph, rpl, p.v8 != 0, rr); else ld4_planes(rph, rpl, rr);
    }
}
// (2) scale / residual / bias / ReLU of the staged accumulator values (a0, a1), then the fp32 value (and its tf32 `lo` companion when asked)
// and / or the fp16 (hi, lo) planes the next tensor-core conv reads.  Returns the largest magnitude written to fp16 planes (fp16-range guard).
__device__ __forceinline__ float tcp_epi_out(const TcParams& p, long long pix, int n, const float4& a0, const float4& a1, const float (&rr)[8]) {
    const bool full8 = n + 8 <= p.Cout;
    const float osc = p.out_scale;
    float amax = 0.f;
    const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
    float a[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) a[k] = av[k] * osc + rr[k];
    if (p.bias) {
        if (full8) {
            float bb[8];
            ld8(p.bias + n, bb);
#pragma unroll
            for (int k = 0; k < 8; ++k) a[k] += bb[k];
        } else {
            const float4 b4 = ldg4(p.bias + n);
            a[0] += b4.x; a[1] += b4.y; a[2] += b4.z; a[3] += b4.w;
        }
    }
    if (p.relu) {
#pragma unroll
        for (int k = 0; k < 8; ++k) a[k] = fmaxf(a[k], 0.f);
    }
    if (p.out) {      // (nullptr: planes-only output, no fp32 copy is written)
        float* op = p.out + pix * p.out_cs + p.out_co + n;
        if (full8) st8(op, a);
        else *reinterpret_cast<float4*>(op) = make_float4(a[0], a[1], a[2], a[3]);
    }
    if (p.out_lo) {   // tf32 companion for the next 3xTF32 conv: the part of the value the MMA does not see
        float* olo = p.out_lo + pix * p.out_cs + p.out_co + n;
        float l[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) l[k] = a[k] - __uint_as_float(__float_as_uint(a[k]) & 0xFFFFE000u);
        if (full8) st8(olo, l);
        else *reinterpret_cast<float4*>(olo) = make_float4(l[0], l[1], l[2], l[3]);
    }
    if (p.out_h16_hi) {      // fp16 hi/lo planes for the next fp16-split conv
        __half* oh = reinterpret_cast<__half*>(p.out_h16_hi) + pix * p.out_cs + p.out_co + n;
        __half* ol16 = reinterpret_cast<__half*>(p.out_h16_lo) + pix * p.out_cs + p.out_co + n;
        uint2 h0, l0, h1, l1;
#pragma unroll
        for (int k = 0; k < 8; ++k) amax = fmaxf(amax, fabsf(a[k]));     // (in the Cout % 8 == 4 tail a[4..7] belong to zero-weight padding columns)
        split4(a, h0, l0);
        if (full8) {
            split4(a + 4, h1, l1);
            if (p.v8) {
                *reinterpret_cast<uint4*>(oh) = make_uint4(h0.x, h0.y, h1.x, h1.y);
                *reinterpret_cast<uint4*>(ol16) = make_uint4(l0.x, l0.y, l1.x, l1.y);
            } else {
                *reinterpret_cast<uint2*>(oh) = h0; *reinterpret_cast<uint2*>(oh + 4) = h1;
                *reinterpret_cast<uint2*>(ol16) = l0; *reinterpret_cast<uint2*>(ol16 + 4) = l1;
            }
        } else {
            *reinterpret_cast<uint2*>(oh) = h0;
            *reinterpret_cast<uint2*>(ol16) = l0;
        }
    }
    return amax;
}

// Epilogue of one tile run by the 256 consumer threads (dcn_fused.cu) after the tile's accumulator has been staged in shared memory ([128][ld]
// fp32, row = tile pixel): thread (warp, lane) owns pixel row 32 (warp % 4) + lane and column half warp / 4.  Returns the largest magnitude
// written to fp16 planes.  `swz`: the staged tile's chunk swizzle (wg_stage).
template <int N>
__device__ __forceinline__ float tcp_store_tile(const TcParams& p, const float* tile, int ld, int u, int mt_units, int warp, int lane, int swz = 0) {
    constexpr int HALF = ((N + 31) / 32) * 16;                     // accumulator columns per thread
    const int q = warp & 3, half = warp >> 2;
    const int cb = half * HALF;
    int mu, nt;
    unit_tile(p, u, mt_units, mu, nt);
    const int ncols = min(HALF, min(p.BN, p.cout_pad - nt * p.BN) - cb);      // valid columns of this thread in this tile (<= 0: none)
    const TcGeom g = tile_geom(p, mu);
    const int r = q * 32 + lane;
    const int ho = g.h0 + r / TC_TW, wo = g.w0 + r % TC_TW;
    float amax = 0.f;
    if (!tcp_stores(p, g, ho, wo) || ncols <= 0 || (p.dbg & 16)) return amax;
    const long long pix = tcp_out_pix(g, ho, wo);
    const long long rpix = tcp_res_pix(g, ho, wo);
    const float* acc = tile + r * ld;
    int sw = r & swz;
    if (swz) asm volatile("" : "+r"(sw));                           // (as in wg_stage)
    const int nbase = nt * p.BN + cb;
#pragma unroll
    for (int col = 0; col < HALF; col += 8) {
        const int n = nbase + col;
        if (col < ncols && n + 4 <= p.Cout) {
            float rr[8];
            tcp_epi_res(p, rpix, n, rr);
            const int j = (cb + col) >> 2;                       // 16-byte chunk of the staged row
            const float4 a0 = *reinterpret_cast<const float4*>(acc + ((j ^ sw) << 2)), a1 = *reinterpret_cast<const float4*>(acc + (((j + 1) ^ sw) << 2));
            amax = fmaxf(amax, tcp_epi_out(p, pix, n, a0, a1, rr));
        }
    }
    return amax;
}

// VD3D_PDL=1: the persistent tensor-core kernels are launched as programmatic dependents of their predecessor in the stream (pdl_wait() in the kernels)
inline bool pdl_enabled() {
    static int v = -1;
    if (v < 0) { const char* e = getenv("VD3D_PDL"); v = (e && atoi(e) != 0) ? 1 : 0; }
    return v == 1;
}

// Launch of a tensor-core kernel: `threads` per CTA, `smem` bytes of dynamic shared memory (the first launch of each kernel raises its limit to
// 227 KB), as a programmatic dependent of its predecessor when pdl_enabled().
template <auto Kernel, class... Args>
inline cudaError_t tc_launch(int grid, int threads, size_t smem, void* stream, const Args&... args) {
    static bool attr_set = false;
    if (!attr_set) {
        const cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
        if (e != cudaSuccess) return e;
        attr_set = true;
    }
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3((unsigned)grid); cfg.blockDim = dim3((unsigned)threads); cfg.dynamicSmemBytes = smem; cfg.stream = (cudaStream_t)stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, Kernel, args...);
}

inline int make_map_wgt(CUtensorMap* m, const void* base, int Cout, int K, int BN, int esize = 4, int rowb = 128) {
    EncodeTiledFn enc = get_encode();
    if (!enc) { set_error("conv2d_tc: cuTensorMapEncodeTiled unavailable"); return VD3D_ECUDA; }
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)Cout};
    cuuint64_t strides[1] = {(cuuint64_t)K * esize};
    cuuint32_t box[2] = {(cuuint32_t)(rowb / esize), (cuuint32_t)BN};
    cuuint32_t es[2] = {1, 1};
    CUresult r = enc(m, esize == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     rowb == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("conv2d_tc: cuTensorMapEncodeTiled(weights) failed: %d", (int)r); return VD3D_ECUDA; }
    return VD3D_OK;
}

// The row-strip kernel (conv2d_row64.cu) runs a conv of the fp16-split engine bit-identically to conv2d_tcp_kernel when it is a 3x3 / stride-1 /
// pad-1 conv over at most 64 input channels into one output tile of at most 64 columns, with a plain (fp32 or plane) residual or none.
inline bool conv2d_row64_eligible(const TcParams& p) {
    return p.f16 && p.passes == 3 && !p.two_pass && p.KH == 3 && p.KW == 3 && p.stride == 1 && p.pad == 1 && p.dil == 1 && p.stride_w == 1 &&
           p.pad_w == 1 && p.cin_pad == 64 && p.BN <= 64 && p.n_tiles == 1 && p.n_levels == 0 && p.res_up_W == 0 && !p.pool_out && !p.out_lo;
}
int conv2d_row64_launch(TcParams& p, const void* in_hi, const void* in_lo, int in_cs, int in_co, const void* w_hi, const void* w_lo, void* stream);


}  // namespace vd3d
