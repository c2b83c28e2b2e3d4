// Fused (modulated) deformable convolution on the tensor cores: the bilinear gather of deformable im2col goes STRAIGHT into the swizzled
// shared-memory A operand of the wgmma GEMM.  The reference writes `columns[C*9, H*W]` to HBM per image and reads it back with cuBLAS
// (R/lib/ops/dcn/src/cuda/deform_conv_cuda.cpp:539-556, kernel deform_conv_cuda_kernel.cu:570-633); round 1 of this repo still wrote the
// fp16 (hi, lo) column planes (4 x 9C bytes per pixel) and re-read them in a 1x1 conv.  Here no column tensor exists:
//
//   out[pix, o] = bias[o] + sum_{tap, c} W[o, tap*C + c] * mask[pix, tap] * bilinear(x[.., c], p(pix, tap))
//
//   HBM traffic per layer = x (read once; the 36 (tap, corner) re-reads of a pixel are L1 / L2 hits inside a spatial 8 x 16 tile)
//                           + offsets / mask + output, instead of + 2 x 36 C bytes per pixel of column planes.
//
// Structure = the persistent conv kernel (conv2d_tc.cu) with the activation TMA producer replaced by eight GATHER warps:
//   warps 0..7  two consumer warpgroups: 3 kind::f16 MMAs per K step on (A_lo W_hi + A_hi W_lo + A_hi W_hi), chunked promotion, then the
//               epilogue (tcp_store_tile of tc_conv.cuh: scale / bias / residual / ReLU -> fp32 and / or fp16 planes)
//   warp 8      weight producer: TMA boxes [64 k][BN] of the (hi, lo) weight matrix, one per k-block (tap, 64-channel chunk)
//   warps 9..16 gather: per tile the sampling position, validity and the 4 bilinear weights of every (pixel, tap) are computed once into
//               shared memory (same rule as dcn.cu: a tap contributes iff h > -1, w > -1, h < H, w < W; corners are individually zero
//               outside); per k-block each thread produces 8 channels of 4 pixels: 4 corner loads of 32 B, the weighted sum, x mask,
//               the (hi, lo) fp16 split, and two 16-byte stores into the SWIZZLE_128B K-major operand layout
//               (row m = pixel, 16-byte chunk j at ((m / 8) * 1024 + (m % 8) * 128 + ((j ^ (m % 8)) * 16)), then fence.proxy.async and an
//               mbarrier arrive: the tensor core reads the stage through its descriptor like a TMA-written one.
// K order = tap-major, 64-channel chunks inside, promotion every `chunk` k-blocks: exactly the order of the unfused path (im2col planes ->
// 1x1 conv), and the gather arithmetic is the same explicit fma chain, so both paths produce identical bits (tests assert torch.equal).
#include "tc_conv.cuh"
#include <cstring>

namespace vd3d {

constexpr int DF_THREADS = 256 + 32 + 256;      // consumers, weight producer, gather warps
constexpr int DF_GATHER0 = 288;                  // first gather thread
constexpr int DF_GATHER_WARPS = 8;
constexpr int DF_MAXK = 9;

struct DfParams {
    const float* x; int H, W, C, x_cs, x_co;        // input NHWC fp32 [B][H][W][x_cs]
    const float* om; int om_cs, off_co, msk_co;     // offsets (channel off_co + 2k = dh, +1 = dw) and mask (msk_co + k), NHWC at OUTPUT resolution
    int has_mask, mask_sigmoid;
    int KW, stride, pad, dil;
    int K;                                          // taps
    int cchunks;                                    // C / 64
    int stages;                                     // operand ring (fused kernel) / weight ring (staged kernel)
    uint32_t stage_bytes;
    int dbg;                                        // timing knock-outs (VD3D_DF_DEBUG; results wrong): 1 no corner loads, 2 no offset / mask loads, 4 no operand stores, 8 one MMA per k-block
};

struct DfSample { int base_flags; float w1, w2, w3, w4, m; };      // base + W + 1 in bits 0..25, validity bits 26..30 (bit 30 = tap inside)

template <int BN>
__global__ void __launch_bounds__(DF_THREADS, 1)
deform_conv_fused_kernel(const __grid_constant__ CUtensorMap mapWhi, const __grid_constant__ CUtensorMap mapWlo, const TcParams p, const DfParams q) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    constexpr int LD = BN + 4;
    const uint32_t a_bytes = 128u * 128u;                        // one A plane of a stage: 128 pixels x 64 fp16
    const uint32_t b_bytes = (uint32_t)BN * 128u;
    const uint32_t stage_bytes = q.stage_bytes;                  // [A hi | A lo | W hi | W lo]
    DfSample* samp = reinterpret_cast<DfSample*>(smem + (size_t)q.stages * stage_bytes);          // [128][K]
    float* tile = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(samp) + sizeof(DfSample) * 128 * DF_MAXK);     // [128][LD] staged accumulator
    uint64_t* bars = reinterpret_cast<uint64_t*>(tile + 128 * LD);
    uint64_t* fullA = bars;                       // [stages]  gather warps -> consumers (8 arrivals)
    uint64_t* fullB = fullA + q.stages;           // [stages]  TMA -> consumers
    uint64_t* empty = fullB + q.stages;           // [stages]  consumers (8 warps) -> producers

    const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
    const int KB = q.K * q.cchunks;
    const int mt_units = p.m_tiles;
    const int units = mt_units * p.n_tiles;
    const int u0 = (int)blockIdx.x, ustep = (int)gridDim.x;

    if (threadIdx.x == 0) {
        for (int s = 0; s < q.stages; ++s) { mbar_init(&fullA[s], DF_GATHER_WARPS); mbar_init(&fullB[s], 1); mbar_init(&empty[s], 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 8) {
        // ================= weight producer =================
        int it = 0;
        for (int u = u0; u < units; u += ustep) {
            const int nt = unit_nt(p, u, mt_units);
            const int n0 = nt * BN;
            for (int kb = 0; kb < KB; ++kb, ++it) {
                const int s = it % q.stages, ph = (it / q.stages) & 1;
                mbar_wait(&empty[s], ph ^ 1);
                if (elect_one()) {
                    uint8_t* st = smem + (size_t)s * stage_bytes + 2 * a_bytes;
                    mbar_expect_tx(&fullB[s], 2u * b_bytes);
                    tma_load_2d(st, &mapWhi, &fullB[s], kb * 64, n0);              // K column of k-block kb = (tap * cchunks + chunk) * 64
                    tma_load_2d(st + b_bytes, &mapWlo, &fullB[s], kb * 64, n0);
                }
                __syncwarp();
            }
        }
    } else if (warp < 8) {
        // ================= consumer warpgroups =================
        const int wg = warp >> 2;
        const int mode = (q.dbg & 8) ? 1 : 0;
        int it = 0;
        auto acquire = [&]() {
            const int s = it % q.stages, ph = (it / q.stages) & 1;
            mbar_wait(&fullB[s], ph);
            mbar_wait(&fullA[s], ph);
            const uint32_t sa = smem_u32(smem + (size_t)s * stage_bytes);
            const uint32_t aw = sa + (uint32_t)wg * 64u * 128u;
            ++it;
            return KbOperands{make_sdesc(aw), make_sdesc(aw + a_bytes), make_sdesc(sa + 2 * a_bytes), make_sdesc(sa + 2 * a_bytes + b_bytes), s};
        };
        auto release = [&](int st) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[st]);
        };
        auto issued = [] {};
        float tot[BN / 2], c[BN / 2];
        float amax = 0.f;
        for (int u = u0; u < units; u += ustep) {
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) tot[i] = 0.f;
            // small terms first (same MMA order and chunking as conv2d_tcp_kernel)
            if (mode == 0) wg_tile_kloop<BN, true, 0, 4>(tot, c, KB, p.chunk, acquire, release, issued);
            else wg_tile_kloop<BN, true, 1, 4>(tot, c, KB, p.chunk, acquire, release, issued);
            consumers_sync();
            wg_stage<BN>(tot, tile, LD, wg, warp, lane);
            consumers_sync();
            amax = fmaxf(amax, tcp_store_tile<BN>(p, tile, LD, u, mt_units, warp, lane));
        }
        note_fp16_range(amax, p.range_flag);
    } else {
        // ================= gather warps (256 threads) =================
        const int gt = (int)threadIdx.x - DF_GATHER0;     // 0..255
        const int j = gt & 7;                             // 8-channel group inside the 64-channel chunk
        const int m0 = gt >> 3;                           // pixels m0, m0 + 32, m0 + 64, m0 + 96 of the tile
        int it = 0;
        for (int u = u0; u < units; u += ustep) {
            int mu, nt;
            unit_tile(p, u, mt_units, mu, nt);
            int mt = mu;
            const int tw = mt % p.tiles_w; mt /= p.tiles_w;
            const int th = mt % p.tiles_h; const int b = mt / p.tiles_h;
            // ---- sampling table of the tile: one entry per (pixel, tap) ----
            asm volatile("bar.sync 1, 256;" ::: "memory");         // every gather thread is done with the previous tile's table
            for (int i = gt; i < 128 * q.K; i += 256) {
                const int m = i / q.K, k = i - m * q.K;
                const int ho = th * TC_TH + m / TC_TW, wo = tw * TC_TW + m % TC_TW;
                DfSample sm;
                sm.base_flags = 0; sm.w1 = sm.w2 = sm.w3 = sm.w4 = 0.f; sm.m = 1.f;
                if (ho < p.Ho && wo < p.Wo) {
                    const long long pix = ((long long)b * p.Ho + ho) * p.Wo + wo;
                    const int kh = k / q.KW, kw = k - kh * q.KW;
                    const float* op = q.om + pix * q.om_cs + q.off_co + 2 * k;
                    const float dh = __ldg(op), dw = __ldg(op + 1);
                    if (q.has_mask) {
                        float mv = __ldg(q.om + pix * q.om_cs + q.msk_co + k);
                        if (q.mask_sigmoid) mv = __fdiv_rn(1.0f, 1.0f + expf(-mv));
                        sm.m = mv;
                    }
                    const float h = (float)(ho * q.stride - q.pad + kh * q.dil) + dh;
                    const float w = (float)(wo * q.stride - q.pad + kw * q.dil) + dw;
                    if (h > -1.f && w > -1.f && h < (float)q.H && w < (float)q.W) {
                        const int hl = (int)floorf(h), wl = (int)floorf(w);
                        const float lh = h - (float)hl, lw = w - (float)wl, hh = 1.f - lh, hw = 1.f - lw;
                        int flags = 16;
                        if (hl >= 0 && wl >= 0) flags |= 1;
                        if (hl >= 0 && wl + 1 <= q.W - 1) flags |= 2;
                        if (hl + 1 <= q.H - 1 && wl >= 0) flags |= 4;
                        if (hl + 1 <= q.H - 1 && wl + 1 <= q.W - 1) flags |= 8;
                        sm.base_flags = (hl * q.W + wl + q.W + 1) | (flags << 26);
                        sm.w1 = hh * hw; sm.w2 = hh * lw; sm.w3 = lh * hw; sm.w4 = lh * lw;
                    }
                }
                samp[i] = sm;
            }
            asm volatile("bar.sync 1, 256;" ::: "memory");
            const float* xb = q.x + ((long long)b * q.H * q.W) * q.x_cs + q.x_co;
            for (int kb = 0; kb < KB; ++kb, ++it) {
                const int tap = kb / q.cchunks, ch = kb - tap * q.cchunks;
                const int s = it % q.stages, ph = (it / q.stages) & 1;
                mbar_wait(&empty[s], ph ^ 1);
                uint8_t* sa = smem + (size_t)s * stage_bytes;
                const int c = ch * 64 + j * 8;
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    const int m = m0 + 32 * r;
                    const DfSample sm = samp[m * q.K + tap];
                    float a[8];
#pragma unroll
                    for (int e = 0; e < 8; ++e) a[e] = 0.f;
                    const int flags = sm.base_flags >> 26;
                    if (flags & 16) {
                        const int base = (sm.base_flags & 0x3FFFFFF) - q.W - 1;
                        const float* x1 = xb + (long long)base * q.x_cs + c;
                        const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
                        const float4 v1a = (flags & 1) ? ldg4(x1) : z, v1b = (flags & 1) ? ldg4(x1 + 4) : z;
                        const float4 v2a = (flags & 2) ? ldg4(x1 + q.x_cs) : z, v2b = (flags & 2) ? ldg4(x1 + q.x_cs + 4) : z;
                        const float4 v3a = (flags & 4) ? ldg4(x1 + (long long)q.W * q.x_cs) : z, v3b = (flags & 4) ? ldg4(x1 + (long long)q.W * q.x_cs + 4) : z;
                        const float4 v4a = (flags & 8) ? ldg4(x1 + (long long)(q.W + 1) * q.x_cs) : z, v4b = (flags & 8) ? ldg4(x1 + (long long)(q.W + 1) * q.x_cs + 4) : z;
#define VD3D_DF_MIX(o, f) a[o] = __fmul_rn(fmaf(sm.w4, v4##f, fmaf(sm.w3, v3##f, fmaf(sm.w2, v2##f, __fmul_rn(sm.w1, v1##f)))), sm.m)
                        VD3D_DF_MIX(0, a.x); VD3D_DF_MIX(1, a.y); VD3D_DF_MIX(2, a.z); VD3D_DF_MIX(3, a.w);
                        VD3D_DF_MIX(4, b.x); VD3D_DF_MIX(5, b.y); VD3D_DF_MIX(6, b.z); VD3D_DF_MIX(7, b.w);
#undef VD3D_DF_MIX
                    }
                    uint2 h0, l0, h1, l1;
                    split4(a, h0, l0);
                    split4(a + 4, h1, l1);
                    const uint32_t off = (uint32_t)(m >> 3) * 1024u + (uint32_t)(m & 7) * 128u + (uint32_t)((j ^ (m & 7)) * 16);
                    *reinterpret_cast<uint4*>(sa + off) = make_uint4(h0.x, h0.y, h1.x, h1.y);
                    *reinterpret_cast<uint4*>(sa + a_bytes + off) = make_uint4(l0.x, l0.y, l1.x, l1.y);
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic-proxy writes -> visible to the tensor core's async-proxy reads
                __syncwarp();
                if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&fullA[s])) : "memory");
            }
        }
    }
}

// ----------------------------------------------------------------------------------------------------------------
// Staged form (3x3, stride 1, pad 1, dilation 1: every deformable layer of the DLA up-sampling path and of the Yolo3D head).
// The gather warps of the kernel above read the four bilinear corners of every (pixel, tap) from global memory: 36 loads per output
// value whose latency eight warps cannot hide.  Here the input neighbourhood of the tile is STAGED IN SHARED MEMORY by TMA, once per
// (tile, 64-channel chunk):
//   region = rows [h0 - 2, h0 + 10) x columns [w0 - 2, w0 + 18) x 64 channels of x (fp32, 61,440 B; out-of-image pixels are zero-filled by
//   the TMA unit, which is exactly the reference's "corner outside the image contributes zero" rule);
//   the nine taps of the chunk then gather from shared memory (a corner that falls outside the staged region -- an offset beyond
//   +-1 pixel around the regular tap position -- is read from global memory instead: correct for any offset, fast for small ones).
// The sampling table (position, validity, 4 weights, mask of every (pixel, tap)) is computed once per tile for all nine taps.
// Weights run through their own TMA ring (up to 4 deep, as many 16 KB blocks as shared memory leaves), the gathered operand through a
// 2-deep ring: with one shared 2-deep ring every k-block pays the full latency of its weight load.
// Each gather thread owns channels [4j, 4j + 4) and [32 + 4j, 32 + 4j + 4) of four pixels: its two 16-byte shared-memory reads per corner
// are conflict-free (8 lanes = 128 contiguous bytes).
// K order: 64-channel chunk outermost, taps inside (k = (chunk * 9 + tap) * 64 + c): the weight matrix and the unfused A/B path
// (vd3d_deform_im2col_h16 with k_order = 1) use the same order, so both still produce identical bits.
// Shared memory: A ring 2 x 32 KB + W ring + region 60 KB + sample table 31.5 KB + staged accumulator 34 KB (BN = 64: 2 W stages, 222 KB).
// ----------------------------------------------------------------------------------------------------------------
constexpr int DFS_HALO = 2;
constexpr int DFS_RH = TC_TH + 2 * DFS_HALO, DFS_RW = TC_TW + 2 * DFS_HALO;       // 12 x 20 pixels
constexpr uint32_t DFS_REGION_BYTES = DFS_RH * DFS_RW * 64 * 4;                   // 61,440
constexpr int DFS_A_STAGES = 2, DFS_W_STAGES = 4;      // (W: at most)
constexpr uint32_t DFS_A_STAGE = 2u * 128u * 128u;                                 // A hi | A lo

struct DfSample2 { int hl, wl_flags; float w1, w2, w3, w4, m; };                  // wl in the low 16 bits (biased by 16384), validity bits 16..20

template <int BN>
__global__ void __launch_bounds__(DF_THREADS, 1)
deform_conv_fused_staged_kernel(const __grid_constant__ CUtensorMap mapX, const __grid_constant__ CUtensorMap mapWhi,
                                const __grid_constant__ CUtensorMap mapWlo, const TcParams p, const DfParams q) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    constexpr int LD = BN + 4;
    const uint32_t a_bytes = 128u * 128u;
    const uint32_t b_bytes = (uint32_t)BN * 128u;
    const uint32_t w_stage = 2u * b_bytes;
    const int WS = q.stages;                       // weight ring depth
    uint8_t* smemA = smem;
    uint8_t* smemW = smemA + (size_t)DFS_A_STAGES * DFS_A_STAGE;
    uint8_t* region = smemW + (size_t)WS * w_stage;
    DfSample2* samp = reinterpret_cast<DfSample2*>(region + DFS_REGION_BYTES);               // [K taps][128 pixels]
    float* tile = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(samp) + (size_t)DF_MAXK * 128 * sizeof(DfSample2));     // [128][LD]
    uint64_t* bars = reinterpret_cast<uint64_t*>(tile + 128 * LD);
    uint64_t* fullA = bars;                        // [2]  gather warps -> consumers (8 arrivals)
    uint64_t* emptyA = fullA + DFS_A_STAGES;       // [2]  consumers (8 warps) -> gather warps
    uint64_t* fullW = emptyA + DFS_A_STAGES;       // [WS] weight TMA -> consumers
    uint64_t* emptyW = fullW + WS;                 // [WS] consumers (8 warps) -> weight producer
    uint64_t* fullR = emptyW + WS;                 // [1]  region TMA -> gather warps
    uint64_t* emptyR = fullR + 1;                  // [1]  gather warps -> region producer (8 arrivals)

    const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
    const int KB = q.K * q.cchunks;
    const int mt_units = p.m_tiles;
    const int units = mt_units * p.n_tiles;
    const int u0 = (int)blockIdx.x, ustep = (int)gridDim.x;

    if (threadIdx.x == 0) {
        for (int s = 0; s < DFS_A_STAGES; ++s) { mbar_init(&fullA[s], DF_GATHER_WARPS); mbar_init(&emptyA[s], 8); }
        for (int s = 0; s < WS; ++s) { mbar_init(&fullW[s], 1); mbar_init(&emptyW[s], 8); }
        mbar_init(fullR, 1); mbar_init(emptyR, DF_GATHER_WARPS);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 8) {
        // ================= TMA producer: the input region of every (tile, chunk), then its nine weight blocks =================
        int itw = 0, ir = 0;
        for (int u = u0; u < units; u += ustep) {
            int mu, nt;
            unit_tile(p, u, mt_units, mu, nt);
            int mt = mu;
            const int tw = mt % p.tiles_w; mt /= p.tiles_w;
            const int th = mt % p.tiles_h; const int b = mt / p.tiles_h;
            const int n0 = nt * BN;
            for (int ch = 0; ch < q.cchunks; ++ch, ++ir) {
                mbar_wait(emptyR, (ir & 1) ^ 1);                     // the gather warps are done with the previous region
                if (elect_one()) {
                    mbar_expect_tx(fullR, DFS_REGION_BYTES);
                    tma_load_4d(region, &mapX, fullR, ch * 64, tw * TC_TW - DFS_HALO, th * TC_TH - DFS_HALO, b);
                }
                __syncwarp();
                for (int t = 0; t < q.K; ++t, ++itw) {
                    const int s = itw % WS, ph = (itw / WS) & 1;
                    mbar_wait(&emptyW[s], ph ^ 1);
                    if (elect_one()) {
                        uint8_t* st = smemW + (size_t)s * w_stage;
                        mbar_expect_tx(&fullW[s], w_stage);
                        const int kcol = (ch * q.K + t) * 64;
                        tma_load_2d(st, &mapWhi, &fullW[s], kcol, n0);
                        tma_load_2d(st + b_bytes, &mapWlo, &fullW[s], kcol, n0);
                    }
                    __syncwarp();
                }
            }
        }
    } else if (warp < 8) {
        // ================= consumer warpgroups =================
        const int wg = warp >> 2;
        const int mode = (q.dbg & 8) ? 1 : 0;
        int it = 0;
        auto acquire = [&]() {
            const int sa = it % DFS_A_STAGES, pa = (it / DFS_A_STAGES) & 1;
            const int sw = it % WS, pw = (it / WS) & 1;
            mbar_wait(&fullW[sw], pw);
            mbar_wait(&fullA[sa], pa);
            const uint32_t aa = smem_u32(smemA + (size_t)sa * DFS_A_STAGE) + (uint32_t)wg * 64u * 128u, ww = smem_u32(smemW + (size_t)sw * w_stage);
            return KbOperands{make_sdesc(aa), make_sdesc(aa + a_bytes), make_sdesc(ww), make_sdesc(ww + b_bytes), it++};
        };
        auto release = [&](int i) {
            __syncwarp();
            if (lane == 0) { mbar_arrive(&emptyA[i % DFS_A_STAGES]); mbar_arrive(&emptyW[i % WS]); }
        };
        auto issued = [] {};
        float tot[BN / 2], c[BN / 2];
        float amax = 0.f;
        for (int u = u0; u < units; u += ustep) {
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) tot[i] = 0.f;
            if (mode == 0) wg_tile_kloop<BN, true, 0, 4>(tot, c, KB, p.chunk, acquire, release, issued);
            else wg_tile_kloop<BN, true, 1, 4>(tot, c, KB, p.chunk, acquire, release, issued);
            consumers_sync();
            wg_stage<BN>(tot, tile, LD, wg, warp, lane);
            consumers_sync();
            amax = fmaxf(amax, tcp_store_tile<BN>(p, tile, LD, u, mt_units, warp, lane));
        }
        note_fp16_range(amax, p.range_flag);
    } else {
        // ================= gather warps (256 threads) =================
        const int gt = (int)threadIdx.x - DF_GATHER0;
        const int j = gt & 7;                             // channel groups [4j, 4j + 4) and [32 + 4j, 32 + 4j + 4) of the chunk
        const int m0 = gt >> 3;                           // pixels m0, m0 + 32, m0 + 64, m0 + 96 of the tile
        int it = 0, ir = 0;
        for (int u = u0; u < units; u += ustep) {
            int mu, nt;
            unit_tile(p, u, mt_units, mu, nt);
            int mt = mu;
            const int tw = mt % p.tiles_w; mt /= p.tiles_w;
            const int th = mt % p.tiles_h; const int b = mt / p.tiles_h;
            const int rh0 = th * TC_TH - DFS_HALO, rw0 = tw * TC_TW - DFS_HALO;           // image coordinates of region pixel (0, 0)
            const float* xb = q.x + ((long long)b * q.H * q.W) * q.x_cs + q.x_co;
            // ---- sampling table of the tile, all taps: entry [tap][pixel] ----
            asm volatile("bar.sync 1, 256;" ::: "memory");         // every gather thread is done with the previous tile's table
            for (int i = gt; i < 128 * q.K; i += 256) {
                const int tap = i >> 7, m = i & 127;
                const int ho = th * TC_TH + m / TC_TW, wo = tw * TC_TW + m % TC_TW;
                DfSample2 sm;
                sm.hl = 0; sm.wl_flags = 0; sm.w1 = sm.w2 = sm.w3 = sm.w4 = 0.f; sm.m = 1.f;
                if (ho < p.Ho && wo < p.Wo) {
                    const long long pix = ((long long)b * p.Ho + ho) * p.Wo + wo;
                    const int kh = tap / q.KW, kw = tap - kh * q.KW;
                    const float* op = q.om + pix * q.om_cs + q.off_co + 2 * tap;
                    float dh = 0.25f, dw = 0.25f;
                    if (!(q.dbg & 2)) { dh = __ldg(op); dw = __ldg(op + 1); }
                    if (q.has_mask && !(q.dbg & 2)) {
                        float mv = __ldg(q.om + pix * q.om_cs + q.msk_co + tap);
                        if (q.mask_sigmoid) mv = __fdiv_rn(1.0f, 1.0f + expf(-mv));
                        sm.m = mv;
                    }
                    const float h = (float)(ho * q.stride - q.pad + kh * q.dil) + dh;
                    const float w = (float)(wo * q.stride - q.pad + kw * q.dil) + dw;
                    if (h > -1.f && w > -1.f && h < (float)q.H && w < (float)q.W) {
                        const int hl = (int)floorf(h), wl = (int)floorf(w);
                        const float lh = h - (float)hl, lw = w - (float)wl, hh = 1.f - lh, hw = 1.f - lw;
                        int flags = 16;
                        if (hl >= 0 && wl >= 0) flags |= 1;
                        if (hl >= 0 && wl + 1 <= q.W - 1) flags |= 2;
                        if (hl + 1 <= q.H - 1 && wl >= 0) flags |= 4;
                        if (hl + 1 <= q.H - 1 && wl + 1 <= q.W - 1) flags |= 8;
                        if (q.dbg & 1) flags = 0;
                        sm.hl = hl; sm.wl_flags = (wl + 16384) | (flags << 16);
                        sm.w1 = hh * hw; sm.w2 = hh * lw; sm.w3 = lh * hw; sm.w4 = lh * lw;
                    }
                }
                samp[i] = sm;
            }
            asm volatile("bar.sync 1, 256;" ::: "memory");
            for (int ch = 0; ch < q.cchunks; ++ch, ++ir) {
                mbar_wait(fullR, ir & 1);
                const float* reg = reinterpret_cast<const float*>(region) + j * 4;
                const int c = ch * 64 + j * 4;
                for (int tap = 0; tap < q.K; ++tap, ++it) {
                    const DfSample2* tb = samp + tap * 128;
                    const int s = it % DFS_A_STAGES, ph = (it / DFS_A_STAGES) & 1;
                    mbar_wait(&emptyA[s], ph ^ 1);
                    uint8_t* sa = smemA + (size_t)s * DFS_A_STAGE;
#pragma unroll
                    for (int r = 0; r < 4; ++r) {
                        const int m = m0 + 32 * r;
                        const DfSample2 sm = tb[m];
                        float a[8];
#pragma unroll
                        for (int e = 0; e < 8; ++e) a[e] = 0.f;
                        const int flags = sm.wl_flags >> 16;
                        if (flags & 16) {
                            const int hl = sm.hl, wl = (sm.wl_flags & 0xFFFF) - 16384;
                            const int hr = hl - rh0, wr = wl - rw0;                        // region coordinates of the top-left corner
                            float4 v[4][2];
#pragma unroll
                            for (int cn = 0; cn < 4; ++cn) {
                                const int dy = cn >> 1, dx = cn & 1;
                                if (flags & (1 << cn)) {
                                    const int y = hr + dy, x = wr + dx;
                                    if ((unsigned)y < (unsigned)DFS_RH && (unsigned)x < (unsigned)DFS_RW) {
                                        const float* sp = reg + (y * DFS_RW + x) * 64;
                                        v[cn][0] = *reinterpret_cast<const float4*>(sp); v[cn][1] = *reinterpret_cast<const float4*>(sp + 32);
                                    } else {                                                // far sample: straight from global memory
                                        const float* gp = xb + ((long long)(hl + dy) * q.W + (wl + dx)) * q.x_cs + c;
                                        v[cn][0] = ldg4(gp); v[cn][1] = ldg4(gp + 32);
                                    }
                                } else {
                                    v[cn][0] = make_float4(0.f, 0.f, 0.f, 0.f); v[cn][1] = v[cn][0];
                                }
                            }
#define VD3D_DF_MIX(o, hf, f) a[o] = __fmul_rn(fmaf(sm.w4, v[3][hf].f, fmaf(sm.w3, v[2][hf].f, fmaf(sm.w2, v[1][hf].f, __fmul_rn(sm.w1, v[0][hf].f)))), sm.m)
                            VD3D_DF_MIX(0, 0, x); VD3D_DF_MIX(1, 0, y); VD3D_DF_MIX(2, 0, z); VD3D_DF_MIX(3, 0, w);
                            VD3D_DF_MIX(4, 1, x); VD3D_DF_MIX(5, 1, y); VD3D_DF_MIX(6, 1, z); VD3D_DF_MIX(7, 1, w);
#undef VD3D_DF_MIX
                        }
                        uint2 h0, l0, h1, l1;
                        split4(a, h0, l0);                                                   // channels 4j .. 4j + 3      -> 16-byte chunk j / 2, half j % 2
                        split4(a + 4, h1, l1);                                               // channels 32 + 4j .. + 3   -> chunk 4 + j / 2
                        if (!(q.dbg & 4)) {
                            const uint32_t row = (uint32_t)(m >> 3) * 1024u + (uint32_t)(m & 7) * 128u, sub = (uint32_t)(j & 1) * 8u;
                            const uint32_t o0 = row + (uint32_t)(((j >> 1) ^ (m & 7)) * 16) + sub, o1 = row + (uint32_t)(((4 + (j >> 1)) ^ (m & 7)) * 16) + sub;
                            *reinterpret_cast<uint2*>(sa + o0) = h0; *reinterpret_cast<uint2*>(sa + o1) = h1;
                            *reinterpret_cast<uint2*>(sa + a_bytes + o0) = l0; *reinterpret_cast<uint2*>(sa + a_bytes + o1) = l1;
                        }
                    }
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    __syncwarp();
                    if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&fullA[s])) : "memory");
                }
                __syncwarp();                                                              // every lane is done reading the region
                if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(emptyR)) : "memory");
            }
        }
    }
}

}  // namespace vd3d

using namespace vd3d;

// sets the shared-memory limit of a kernel instance once, then launches it.  The kernel is a template argument, so each BN instance has
// its own flag: keyed on the kernel's type, the four instances (same signature) would share one, and only the first one launched would get
// the 227 KB limit.
template <auto Kernel, typename... Args>
static cudaError_t df_launch(int grid, size_t smem, void* stream, Args... args) {
    static bool attr_set = false;
    if (!attr_set) {
        const cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
        if (e != cudaSuccess) return e;
        attr_set = true;
    }
    Kernel<<<grid, DF_THREADS, smem, (cudaStream_t)stream>>>(args...);
    return cudaGetLastError();
}

extern "C" int vd3d_deform_conv_fused(const float* x, int B, int H, int W, int C, int x_cs, int x_co,
                                      const float* om, int om_cs, int off_co, int msk_co, int has_mask, int mask_sigmoid,
                                      int KH, int KW, int stride, int pad, int dil, int k_order,
                                      const void* w_hi, const void* w_lo, float out_scale, const float* bias,
                                      const float* res, int res_cs, int res_co,
                                      float* out, void* out_hi16, void* out_lo16, int Cout, int out_cs, int out_co, int relu, void* stream) {
    VD3D_REQUIRE(x && om && w_hi && w_lo && out, "deform_conv_fused: null pointer");
    VD3D_REQUIRE(B > 0 && H > 0 && W > 0 && KH * KW <= DF_MAXK && KH > 0 && KW > 0, "deform_conv_fused: at most 9 taps");
    VD3D_REQUIRE(C % 64 == 0 && x_cs % 4 == 0 && x_co % 4 == 0, "deform_conv_fused: C must be a multiple of 64 (one deformable group)");
    VD3D_REQUIRE(Cout % 4 == 0 && out_cs % 4 == 0 && out_co % 4 == 0, "deform_conv_fused: output channel alignment");
    VD3D_REQUIRE((long long)H * W + W + 1 < (1 << 26), "deform_conv_fused: image too large for the packed sample index");
    VD3D_REQUIRE(!out_hi16 || out_lo16, "deform_conv_fused: fp16 output planes come in (hi, lo) pairs");
    TcParams p;
    memset(&p, 0, sizeof(p));
    DfParams q;
    memset(&q, 0, sizeof(q));
    const int Ho = (H + 2 * pad - (dil * (KH - 1) + 1)) / stride + 1, Wo = (W + 2 * pad - (dil * (KW - 1) + 1)) / stride + 1;
    VD3D_REQUIRE(Ho > 0 && Wo > 0, "deform_conv_fused: empty output");
    const int cp = (Cout + 15) / 16 * 16;
    const int BN = cp <= 64 ? cp : 64;                 // 544 threads leave ~120 registers per thread: 64-column tiles keep the consumers spill-free
    p.B = B; p.H = Ho; p.W = Wo; p.Ho = Ho; p.Wo = Wo; p.Cin = KH * KW * C; p.KH = 1; p.KW = 1; p.stride = 1; p.dil = 1;
    p.Cout = Cout; p.BN = BN; p.passes = 3; p.f16 = 1; p.bk = 64; p.cin_pad = KH * KW * C; p.out_scale = out_scale;
    p.tiles_w = cdiv(Wo, TC_TW); p.tiles_h = cdiv(Ho, TC_TH);
    p.cout_pad = cp; p.m_tiles = p.tiles_w * p.tiles_h * B; p.n_tiles = cdiv(cp, BN);
    p.v8 = (out_cs % 8 == 0 && out_co % 8 == 0 && ((uintptr_t)out & 31) == 0 && (!bias || ((uintptr_t)bias & 31) == 0) &&
            (!res || (res_cs % 8 == 0 && res_co % 8 == 0 && ((uintptr_t)res & 31) == 0)) &&
            (!out_hi16 || ((((uintptr_t)out_hi16 | (uintptr_t)out_lo16) & 15) == 0))) ? 1 : 0;
    p.out_cs = out_cs; p.out_co = out_co; p.res_cs = res_cs; p.res_co = res_co; p.relu = relu;
    p.bias = bias; p.res = res; p.out = out; p.out_h16_hi = out_hi16; p.out_h16_lo = out_lo16;
    p.range_flag = out_hi16 ? fp16_range_flag() : nullptr;
    { const char* e = getenv("VD3D_TC_CHUNK"); p.chunk = e ? atoi(e) : 4; if (p.chunk < 1) p.chunk = 1; }
    { const char* e = getenv("VD3D_TC_DEBUG"); p.dbg = e ? atoi(e) : 0; }
    { const char* e = getenv("VD3D_DF_DEBUG"); q.dbg = e ? atoi(e) : 0; }
    q.x = x; q.H = H; q.W = W; q.C = C; q.x_cs = x_cs; q.x_co = x_co;
    q.om = om; q.om_cs = om_cs; q.off_co = off_co; q.msk_co = msk_co; q.has_mask = has_mask; q.mask_sigmoid = mask_sigmoid;
    q.KW = KW; q.stride = stride; q.pad = pad; q.dil = dil; q.K = KH * KW; q.cchunks = C / 64;
    q.stage_bytes = 2u * 128u * 128u + 2u * (uint32_t)BN * 128u;
    CUtensorMap mWhi, mWlo;
    int rc;
    if ((rc = make_map_wgt(&mWhi, w_hi, Cout, KH * KW * C, BN, 2))) return rc;
    if ((rc = make_map_wgt(&mWlo, w_lo, Cout, KH * KW * C, BN, 2))) return rc;
    const int units = p.m_tiles * p.n_tiles;
    const int grid = units < kNumSMs ? units : kNumSMs;
    const size_t tile_bytes = (size_t)128 * (BN + 4) * sizeof(float);
    const char* es = getenv("VD3D_DCN_STAGED");
    const bool staged = k_order == 1 && stride == 1 && dil == 1 && pad == 1 && KH == 3 && KW == 3 && !(es && atoi(es) == 0);
    if (staged) {
        // input regions through TMA: fp32 NHWC, box {64 c, 20 w, 12 h, 1 b}, no swizzle, zero fill outside the image
        EncodeTiledFn enc = get_encode();
        VD3D_REQUIRE(enc, "deform_conv_fused: cuTensorMapEncodeTiled unavailable");
        CUtensorMap mX;
        cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
        cuuint64_t strides[3] = {(cuuint64_t)x_cs * 4, (cuuint64_t)W * x_cs * 4, (cuuint64_t)H * W * x_cs * 4};
        cuuint32_t box[4] = {64, (cuuint32_t)DFS_RW, (cuuint32_t)DFS_RH, 1};
        cuuint32_t estr[4] = {1, 1, 1, 1};
        CUresult cr = enc(&mX, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void*)(x + x_co), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        VD3D_REQUIRE(cr == CUDA_SUCCESS, "deform_conv_fused: cuTensorMapEncodeTiled(input regions) failed: %d", (int)cr);
        const size_t fixed = (size_t)DFS_A_STAGES * DFS_A_STAGE + (size_t)DFS_REGION_BYTES + (size_t)DF_MAXK * 128 * sizeof(DfSample2) + tile_bytes +
                             32 * sizeof(uint64_t) + 1024;
        int ws = (int)((227 * 1024 - fixed) / (2 * (size_t)BN * 128));
        if (ws > DFS_W_STAGES) ws = DFS_W_STAGES;
        VD3D_REQUIRE(ws >= 2, "deform_conv_fused: shared-memory budget exceeded");
        q.stages = ws;
        const size_t smem = fixed + (size_t)ws * 2 * BN * 128;
        cudaError_t le = cudaErrorInvalidValue;
#define VD3D_DFS_CASE(N) case N: le = df_launch<deform_conv_fused_staged_kernel<N>>(grid, smem, stream, mX, mWhi, mWlo, p, q); break
        switch (BN) { VD3D_DFS_CASE(16); VD3D_DFS_CASE(32); VD3D_DFS_CASE(48); VD3D_DFS_CASE(64); }
#undef VD3D_DFS_CASE
        if (le != cudaSuccess) { set_error("deform_conv_fused_staged: launch failed: %s", cudaGetErrorString(le)); return VD3D_ECUDA; }
        VD3D_CHECK_LAUNCH("deform_conv_fused_staged");
        return VD3D_OK;
    }
    VD3D_REQUIRE(k_order == 0 || C == 64, "deform_conv_fused: the chunk-major K order needs the staged kernel (3x3, stride 1, pad 1, dilation 1)");
    const size_t fixed = sizeof(DfSample) * 128 * DF_MAXK + tile_bytes + 32 * sizeof(uint64_t) + 1024;
    int stages = (int)((227 * 1024 - fixed) / q.stage_bytes);
    if (stages > 6) stages = 6;
    VD3D_REQUIRE(stages >= 2, "deform_conv_fused: tile too large for shared memory");
    q.stages = stages;
    const size_t smem = (size_t)stages * q.stage_bytes + fixed;
    cudaError_t le = cudaErrorInvalidValue;
#define VD3D_DF_CASE(N) case N: le = df_launch<deform_conv_fused_kernel<N>>(grid, smem, stream, mWhi, mWlo, p, q); break
    switch (BN) { VD3D_DF_CASE(16); VD3D_DF_CASE(32); VD3D_DF_CASE(48); VD3D_DF_CASE(64); }
#undef VD3D_DF_CASE
    if (le != cudaSuccess) { set_error("deform_conv_fused: launch failed: %s", cudaGetErrorString(le)); return VD3D_ECUDA; }
    VD3D_CHECK_LAUNCH("deform_conv_fused");
    return VD3D_OK;
}
