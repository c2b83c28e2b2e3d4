// Implicit-GEMM convolution (NHWC activations) on the Hopper tensor cores (wgmma) with fp32-grade accuracy.
//
//   D[m, n] = sum_{tap, c} A[pixel(m) + tap, c] * W[n, tap, c]          M = B*Ho*Wo, N = Cout, K = KH*KW*Cin
//
// * fp16 split (the default engine, vd3d_conv2d_tc16*): every value v is kept as fp16 planes hi = rn16(v), lo = rn16(v - hi); three
//   kind::f16 products per K step (A_lo W_hi + A_hi W_lo + A_hi W_hi) carry 22 significant bits.
//   3xTF32 (vd3d_conv2d_tc): the tensor core reads 32-bit operands and uses their top 19 bits, so every value v is used as v = hi + lo with
//   hi = v & 0xFFFFE000 (what the MMA sees when handed v itself) and lo = v - hi (exact in fp32, kept in a second tensor by the producer);
//   three products A*Whi + Alo*Whi + A*Wlo, the dropped Alo*Wlo term is ~2^-22 relative.
// * No im2col: for k-block (tap, channel chunk) the A operand is ONE 4-D TMA box [chunk][16 w][8 h][1 b] of the input shifted by the tap
//   offset; conv zero padding is TMA out-of-bounds fill.  Swizzled K-major operands (128-byte rows; 64-byte rows for the 32-element stem window).
// * Persistent: one CTA per SM strides over the 128-pixel x BN-channel output tiles (unit_tile: M fastest inside L2-sized M blocks).
//   Warp 8 = TMA producer (one lane) feeding a multi-stage mbarrier ring; warps 0..7 = two consumer warpgroups; warps 9..15 = epilogue
//   (tiles wider than 64 columns, 512 threads; narrower tiles run it on the consumers, tcp_store_tile / tcp_pool_tile, 384 threads).
//   Warpgroup w issues the wgmma of tile rows 64 w .. 64 w + 63 as soon as a stage has landed, keeps one k-block in flight, frees a stage when
//   its MMAs are done, promotes every chunk (wg_promote) and at the end of the tile stages its accumulator in shared memory and hands it to the
//   epilogue warps (tcp_epi_tile), then goes straight on with the next tile's MMAs while the epilogue runs.
// * K order: channel chunk outermost, taps inside, and the same chunking for every tile width: a layer gives bit-identical results
//   whichever tile width the host picks.
#include "tc_conv.cuh"
#include <unordered_map>
#include <string>
#include <cstring>
#include <cstdlib>

namespace vd3d {

// ----------------------------------------------------------------------------------------------------------------
// Epilogue with the 3x3 / stride-2 / pad-1 max-pool fused in (ResNet stem: conv7x7 s2 + BN + ReLU -> MaxPool2d(3, 2, 1), resnet.py:186-189).
// The stem output (64 ch at 1/2 resolution) is by far the largest tensor of the backbone and its only consumer is the pool: here it never
// leaves the SM.  Per 8 x 16 tile: apply scale / bias / ReLU to the staged 128 x 64 accumulator in place, then produce the pooled pixels whose
// 3x3 window touches the tile: 5 x 9 positions.  Positions whose window lies entirely inside the tile (3 of 4 pooled rows, 7 of 8 pooled
// columns) are written with plain stores; the others are shared with the neighbouring tile(s) and combined with atomicMax on the integer bit
// pattern -- exact and order-independent because ReLU makes every value >= +0 (the target rows / columns are zeroed by pool_border_zero_kernel
// before the launch).  max() is exact, so the result equals maxpool(stem) bit for bit.
// ----------------------------------------------------------------------------------------------------------------
constexpr int POOL_LD = 68;          // floats per staged pixel row of the 64-column tile (64 + 4: conflict-free float4 rows)

__device__ __forceinline__ void tcp_pool_tile(const TcParams& p, float* tile, int u, int mt_units, int warp, int lane) {
    const int q = warp & 3, half = warp >> 2;
    const int cb = half * 32;                                        // each thread owns 32 accumulator columns of one pixel
    const float osc = p.out_scale;
    const int et = warp * 32 + lane;                                 // 0..255 among the consumer threads
    int mu, nt;
    unit_tile(p, u, mt_units, mu, nt);
    int mt = mu;
    const int tw = mt % p.tiles_w; mt /= p.tiles_w;
    const int th = mt % p.tiles_h; const int b = mt / p.tiles_h;
    const int r = q * 32 + lane;
    // ---- scale / bias / ReLU, in place in the staged tile ----
    {
        float* tp = tile + r * POOL_LD + cb;
#pragma unroll
        for (int i = 0; i < 32; i += 4) {
            const float4 bb = p.bias ? ldg4(p.bias + cb + i) : make_float4(0.f, 0.f, 0.f, 0.f);
            const float4 v = *reinterpret_cast<const float4*>(tp + i);
            float4 a;
            a.x = fmaxf(v.x * osc + bb.x, 0.f); a.y = fmaxf(v.y * osc + bb.y, 0.f);
            a.z = fmaxf(v.z * osc + bb.z, 0.f); a.w = fmaxf(v.w * osc + bb.w, 0.f);
            *reinterpret_cast<float4*>(tp + i) = a;
        }
    }
    consumers_sync();
    // ---- pooled positions touched by this tile: rows i0 .. i0 + 4, columns j0 .. j0 + 8 ----
    const int h0 = th * TC_TH, w0 = tw * TC_TW, i0 = th * (TC_TH / 2), j0 = tw * (TC_TW / 2);
    for (int item = et; item < 45 * 16; item += TC_CONSUMERS) {
        const int cq = item & 15, pp = item >> 4;
        const int pi = pp / 9, pj = pp - pi * 9;
        const int i = i0 + pi, j = j0 + pj;
        if (i >= p.pool_H || j >= p.pool_W) continue;
        // window rows / columns in tile coordinates, clipped to the tile and to the conv output
        int r_lo = 2 * pi - 1, r_hi = 2 * pi + 1, c_lo = 2 * pj - 1, c_hi = 2 * pj + 1;
        const int r_max = min(TC_TH - 1, p.Ho - 1 - h0), c_max = min(TC_TW - 1, p.Wo - 1 - w0);
        // complete: every window row / column that exists in the conv output lies inside this tile
        const bool complete = (r_lo >= 0 || h0 + r_lo < 0) && (2 * pi <= r_max || h0 + 2 * pi > p.Ho - 1) && (r_hi <= r_max || h0 + r_hi > p.Ho - 1) &&
                              (c_lo >= 0 || w0 + c_lo < 0) && (2 * pj <= c_max || w0 + 2 * pj > p.Wo - 1) && (c_hi <= c_max || w0 + c_hi > p.Wo - 1);
        r_lo = max(r_lo, 0); c_lo = max(c_lo, 0); r_hi = min(r_hi, r_max); c_hi = min(c_hi, c_max);
        if (r_lo > r_hi || c_lo > c_hi) continue;
        float4 m = make_float4(0.f, 0.f, 0.f, 0.f);             // values are >= 0 after the ReLU
        for (int rr = r_lo; rr <= r_hi; ++rr)
            for (int c2 = c_lo; c2 <= c_hi; ++c2) {
                const float4 v = *reinterpret_cast<const float4*>(tile + (rr * TC_TW + c2) * POOL_LD + cq * 4);
                m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
            }
        float* op = p.pool_out + (((long long)b * p.pool_H + i) * p.pool_W + j) * p.pool_cs + p.pool_co + cq * 4;
        if (complete) *reinterpret_cast<float4*>(op) = m;
        else {
            int* ip = reinterpret_cast<int*>(op);
            atomicMax(ip, __float_as_int(m.x)); atomicMax(ip + 1, __float_as_int(m.y));
            atomicMax(ip + 2, __float_as_int(m.z)); atomicMax(ip + 3, __float_as_int(m.w));
        }
    }
}

// zero the pooled positions that receive atomicMax contributions from more than one tile (rows i % 4 == 0, columns j % 8 == 0)
__global__ void pool_border_zero_kernel(float* __restrict__ out, int B, int Hp, int Wp, int C4, int cs, int co) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)B * Hp * Wp * C4;
    if (idx >= total) return;
    const int c4 = (int)(idx % C4); long long r = idx / C4;
    const int j = (int)(r % Wp); r /= Wp;
    const int i = (int)(r % Hp);
    if ((i & 3) != 0 && (j & 7) != 0) return;
    *reinterpret_cast<float4*>(out + (idx / C4) * cs + co + 4 * c4) = make_float4(0.f, 0.f, 0.f, 0.f);
}

// ----------------------------------------------------------------------------------------------------------------
// Persistent kernel.  Shared memory: [stages][A hi | A lo | W hi | W lo] operand ring, the [128][BN + 4] fp32 staged accumulator (unless it is
// staged in the ring: TcParams::tile_in_ring; then rows 64..127 of it when TcParams::split_stage), barriers, the slot log.
//
// Ring slots.  The producer takes the slots round-robin, but passes over the held slot (the stage of a tile's last k-block, where the
// accumulator is staged) while the epilogue has not released it, so the next tile's K loop keeps the other stages flowing, and takes the
// held slot back as soon as it is released (also while it waits for another slot).  The consumers
// cannot predict that order: the producer writes the slot of every k-block into a log of stages + 1 entries, each with a one-arrival
// mbarrier, and the consumers read it before they wait on full[slot].  stages + 1 entries suffice: of any stages + 1 consecutive k-blocks two
// share a slot, so the later one was loaded only after the consumers (or the epilogue, after the consumers staged the tile) released the
// earlier one, and they had read its log entry by then.  Every slot keeps its own phase bit on both sides.
// ----------------------------------------------------------------------------------------------------------------
// row pitch (floats) of the staged accumulator: BN + 4 (conflict-free rows); at BN = 128 unpadded rows with the chunk swizzle of wg_stage,
// so that the 64 KB tile fits in one 64 KB operand stage
__host__ __device__ constexpr int tcp_tile_ld(int BN) { return BN == TC_MAX_BN ? BN : BN + 4; }
// Tiles wider than 64 columns hand their epilogue to the epilogue warps.  Narrower tiles keep it on the consumers (the stem's fused
// max-pool among them): their K loop is short (64 columns: 9 k-blocks of ~890 clocks for a 64-channel 3x3 conv, H100) and the three
// epilogue warps of the 384-thread kernel took longer per tile (~11 k clocks) than the 256 consumer threads, so overlapping made those
// layers slower; on seven warps 64-column tiles measured no faster (DESIGN §4).
__host__ __device__ constexpr bool tcp_epi_warps(int BN) { return BN > 64; }
// Warps 0..7 = consumers, warp 8 = TMA producer, warps 9..15 = epilogue (tiles with epilogue warps: 512 threads; narrower tiles: 384, and
// warps 9..11 leave at once).  ptxas budgets registers per warpgroup at launch: 65536 / 512 = 128 per thread, below the 145 .. 149 the
// 128-column consumers need, so right after the barrier setup the consumer warpgroups raise their budget to TCP_REG_CONSUMER and the
// producer / epilogue warpgroups lower theirs to TCP_REG_EPI (setmaxnreg; 2 x 128 x 160 + 2 x 128 x 96 = 65536).
constexpr int TCP_EPI = 224;
constexpr int TCP_REG_CONSUMER = 160, TCP_REG_EPI = 96;
__host__ __device__ constexpr int tcp_threads(int BN) { return TC_CONSUMERS + 32 + (tcp_epi_warps(BN) ? TCP_EPI : 96); }
static_assert(2 * 128 * TCP_REG_CONSUMER + 2 * 128 * TCP_REG_EPI == 65536, "setmaxnreg split must hand out exactly the register file");
// named barrier of the epilogue warps
__device__ __forceinline__ void epilogue_sync() { asm volatile("bar.sync 3, %0;" ::"n"(TCP_EPI) : "memory"); }

// Epilogue of one staged tile by the epilogue warps (thread et of TCP_EPI).  Item = (pixel row r, 8-column group g), items numbered row-major,
// thread et takes items et, et + TCP_EPI, ...: consecutive lanes cover consecutive column groups of one pixel, so a warp's residual loads and
// output stores are whole runs of a pixel's channels (at BN = 128, 256 contiguous bytes per fp16 plane).  The residual loads of U items are
// issued before the first of them is computed (U x TCP_EPI = 896 item loads in flight per SM).  Per element the arithmetic is that of
// tcp_store_tile.  Covers tile rows r0 .. r1 - 1; row r is read at tile + r * ld.
template <int BN>
__device__ __forceinline__ float tcp_epi_tile(const TcParams& p, const float* tile, int ld, int u, int mt_units, int et, int swz, int r0, int r1) {
    constexpr int CG = BN / 8;                                   // column groups per pixel
    constexpr int U = 4;
    const int ITEMS = r1 * CG;
    int mu, nt;
    unit_tile(p, u, mt_units, mu, nt);
    const int ncols = min(BN, p.cout_pad - nt * BN);              // valid columns of this tile
    const TcGeom geo = tile_geom(p, mu);
    float amax = 0.f;
    if (p.dbg & 16) return amax;
    for (int i0 = r0 * CG + et; i0 < ITEMS; i0 += U * TCP_EPI) {
        float rr[U][8];
        long long pix[U];
        int rg[U];                                               // item = r * CG + g, or -1: nothing to write
#pragma unroll
        for (int i = 0; i < U; ++i) {
            const int idx = i0 + i * TCP_EPI;
            const int r = idx / CG, g = idx - r * CG;
            const int ho = geo.h0 + r / TC_TW, wo = geo.w0 + r % TC_TW;
            const int n = nt * BN + 8 * g;
            rg[i] = (idx < ITEMS && 8 * g < ncols && n + 4 <= p.Cout && tcp_stores(p, geo, ho, wo)) ? idx : -1;
            pix[i] = tcp_out_pix(geo, ho, wo);
            if (rg[i] >= 0) tcp_epi_res(p, tcp_res_pix(geo, ho, wo), n, rr[i]);
        }
#pragma unroll
        for (int i = 0; i < U; ++i) {
            if (rg[i] < 0) continue;
            const int r = rg[i] / CG, g = rg[i] - r * CG;
            const float* acc = tile + r * ld;
            const int sw = r & swz, j = 2 * g;                   // 16-byte chunks j, j + 1 of the staged row (wg_stage's swizzle)
            const float4 a0 = *reinterpret_cast<const float4*>(acc + ((j ^ sw) << 2)), a1 = *reinterpret_cast<const float4*>(acc + (((j + 1) ^ sw) << 2));
            amax = fmaxf(amax, tcp_epi_out(p, pix[i], nt * BN + 8 * g, a0, a1, rr[i]));
        }
    }
    return amax;
}

// activation maps of the levels of a multi-level launch (LV); a one-tensor launch passes the empty form
struct TcLevelMaps { CUtensorMap a[TC_MAX_LEVELS], alo[TC_MAX_LEVELS]; };
struct TcNoLevelMaps { int unused; };

template <int BN, bool F16, bool LV>
__global__ void __launch_bounds__(tcp_threads(BN), 1)
conv2d_tcp_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapAlo,
                  const __grid_constant__ CUtensorMap mapWhi, const __grid_constant__ CUtensorMap mapWlo, const TcParams p,
                  const __grid_constant__ std::conditional_t<LV, TcLevelMaps, TcNoLevelMaps> lmaps) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    constexpr int LD = tcp_tile_ld(BN), swz = BN == TC_MAX_BN ? 7 : 0;
    const bool in_ring = p.tile_in_ring != 0;
    const uint32_t rowb = (uint32_t)p.rowb;                        // 128 (SWIZZLE_128B) or 64 (SWIZZLE_64B)
    const uint32_t a_bytes = 128u * rowb;                          // one A plane of a stage: 128 pixel rows
    const uint32_t b_bytes = (uint32_t)BN * rowb;
    const uint32_t stage_bytes = 2u * a_bytes + 2u * b_bytes;      // [A hi | A lo | W hi | W lo]
    const int kbc = (int)rowb / (F16 ? 2 : 4);                     // channels per k-block
    constexpr bool epi_warps = tcp_epi_warps(BN);
    // (in_ring) split staging: rows 0..63 of the accumulator go to the held stage, rows 64..127 to a separate half tile, so the epilogue can
    // release the stage after the first half
    const bool split = epi_warps && in_ring && p.split_stage != 0;
    float* const tile_sep = reinterpret_cast<float*>(smem + (size_t)p.stages * stage_bytes);      // (tile_in_ring == 0) the tile; (split) rows 64..127
    float* const tile_hi = tile_sep - 64 * LD;                      // (split) row r >= 64 at tile_hi + r * LD
    const int sep_rows = in_ring ? (split ? 64 : 0) : 128;
    uint64_t* full = reinterpret_cast<uint64_t*>(tile_sep + sep_rows * LD);     // [stages]  TMA -> consumers
    uint64_t* empty = full + p.stages;                              // [stages]  consumers (8 warps; the held stage: epilogue warps) -> TMA
    uint64_t* log_bar = empty + p.stages;                           // [stages + 1]  producer -> consumers: slot_log entry written
    uint64_t* acc_full = log_bar + p.stages + 1;                    // consumers (256 threads) -> epilogue: a tile is staged
    uint64_t* acc_empty = acc_full + 1;                             // epilogue -> consumers: the staged tile has been read
    int* mailbox = reinterpret_cast<int*>(acc_empty + 1);           // (in_ring) ring slot of the staged tile
    int* slot_log = mailbox + 1;                                    // [stages + 1]  ring slot of k-block g at entry g % (stages + 1)

    const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0), lane = threadIdx.x & 31;      // (warp-uniform for the compiler)
    const int cchunks = p.cin_pad / kbc;
    const int KB = p.KH * p.KW * cchunks;
    const int u0 = (int)blockIdx.x, ustep = (int)gridDim.x;
    const int mode = tc_mma_mode(p);

    if (threadIdx.x == 0) {
        for (int s = 0; s < p.stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], TC_CONSUMERS / 32); }
        for (int e = 0; e <= p.stages; ++e) mbar_init(&log_bar[e], 1);
        mbar_init(acc_full, TC_CONSUMERS);
        mbar_init(acc_empty, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    pdl_launch_dependents();
    pdl_wait();                            // (PDL launches only) the producer of the activations / residual (and of a tile list) has completed
    // every role reads the same count: the producer, the consumers and the epilogue walk the same units
    const int mt_units = tcp_m_tiles(p);
    const int units = mt_units * p.n_tiles;

    if (warp >= TC_CONSUMERS / 32) {
        // (epilogue-warp tiles) every warp of a warpgroup executes the same setmaxnreg: before the producer / epilogue split
        if constexpr (epi_warps) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(TCP_REG_EPI));
        if (warp > TC_CONSUMERS / 32) {
            // ================= epilogue warps: tile i of this CTA is handed over through acc_full / acc_empty phase i =================
            if (!epi_warps) return;
            const int et = (int)threadIdx.x - (TC_CONSUMERS + 32);
            const bool tr0 = p.trace && blockIdx.x == 0 && et == 0;
            float amax = 0.f;
            int i = 0;
            for (int u = u0; u < units; u += ustep, ++i) {
                const bool tr = tr0 && i < p.trace_n;
                mbar_wait(acc_full, i & 1);
                if (tr) p.trace[7 * p.trace_n + i] = clock64();                                     // [7] epilogue starts
                const int held = *mailbox;
                const float* tile = in_ring ? reinterpret_cast<const float*>(smem + (size_t)held * stage_bytes) : tile_sep;
                // split: the held stage's rows first, then give the stage back and do the rest from the half tile
                for (int part = 0; part < (split ? 2 : 1); ++part) {
                    const bool last = !split || part == 1;
                    amax = fmaxf(amax, tcp_epi_tile<BN>(p, part == 0 ? tile : tile_hi, LD, u, mt_units, et, swz, 64 * part, last ? 128 : 64));
                    // every epilogue thread is done reading the held stage (and the mailbox): give the stage back to the producer (empty[] counts
                    // the 8 consumer warps' arrivals), and at the end the staging buffers to the consumers
                    if (in_ring && part == 0) asm volatile("fence.proxy.async.shared::cta;" ::: "memory");    // generic accesses to the stage before the next TMA write into it
                    epilogue_sync();
                    if (et == 0) {
                        if (in_ring && part == 0) {
                            mbar_arrive(&empty[held], TC_CONSUMERS / 32);
                            if (tr) p.trace[8 * p.trace_n + i] = clock64();                         // [8] stage released
                        }
                        if (last) {
                            mbar_arrive(acc_empty);
                            if (tr) p.trace[11 * p.trace_n + i] = clock64();                        // [11] epilogue done
                        }
                    }
                }
            }
            note_fp16_range(amax, p.range_flag);
        } else {
            if (lane == 0) {
                // ================= TMA producer =================
                const bool lo_too = mode != 1 && !(p.dbg & 2);
                const uint32_t tx = lo_too ? stage_bytes : a_bytes + b_bytes;
                int it = 0, s = 0, i = 0;
                int ph = 0;                                         // bit s: parity of slot s's next fill
                int held = -1;                                      // (in_ring) slot of the latest tile's last k-block, until seen released
                int le = 0;                                         // slot_log entry of k-block it
                for (int u = u0; u < units; u += ustep, ++i) {
                    int skips = 0;
                    int mu, nt;
                    unit_tile(p, u, mt_units, mu, nt);
                    const TcGeom geo = tile_geom(p, mu);
                    const int b = geo.b;
                    const int wi0 = geo.w0 * p.stride_w - geo.pad_w, hi0 = geo.h0 * p.stride - geo.pad_h;
                    const CUtensorMap* mA = &mapA;
                    const CUtensorMap* mAlo = &mapAlo;
                    if constexpr (LV) { mA = &lmaps.a[geo.lvl]; mAlo = &lmaps.alo[geo.lvl]; }
                    const int n0 = nt * BN + geo.w_row;               // (weight rows only: the epilogue's columns are nt * BN ..)
                    int tap = 0, kh = 0, kw = 0, c0 = 0;
                    for (int kb = 0; kb < KB; ++kb, ++it) {
                        int slot = s;
                        if (held < 0) mbar_wait(&empty[s], ((ph >> s) & 1) ^ 1);
                        else {
                            // The epilogue may still be reading the held stage.  Take it as soon as it is released; until then take the next
                            // slot in round-robin order, passing over the held one (the slot after it is not held).
                            const bool at_held = s == held;
                            if (at_held && ++s == p.stages) s = 0;
                            const uint32_t hpar = ((ph >> held) & 1) ^ 1, spar = ((ph >> s) & 1) ^ 1;
                            long long t0 = 0;
                            for (uint32_t spins = 1;; ++spins) {
                                if (mbar_test(&empty[held], hpar)) { slot = held; held = -1; break; }
                                if (mbar_test(&empty[s], spar)) { slot = s; skips += at_held; break; }
                                if ((spins & 0xFFFu) == 0) {                // bounded, as mbar_wait
                                    const long long t = clock64();
                                    if (t0 == 0) t0 = t; else if (t - t0 > 4000000000LL) __trap();
                                }
                            }
                        }
                        if (slot == s && ++s == p.stages) s = 0;
                        ph ^= 1 << slot;
                        const bool tr = p.trace && blockIdx.x == 0 && it < p.trace_n;
                        if (tr) p.trace[it] = clock64();                                          // [0] stage free, about to issue the loads
                        slot_log[le] = slot;
                        mbar_arrive(&log_bar[le]);
                        if (++le > p.stages) le = 0;
                        if (in_ring && kb == KB - 1) held = slot;
                        uint8_t* st = smem + (size_t)slot * stage_bytes;
                        const int wi = wi0 + kw * p.dil, hi = hi0 + kh * p.dil;
                        const int kcol = tap * p.cin_pad + c0;
                        mbar_expect_tx(&full[slot], tx);
                        tma_load_4d(st, mA, &full[slot], c0, wi, hi, b);
                        if (lo_too) tma_load_4d(st + a_bytes, mAlo, &full[slot], c0, wi, hi, b);
                        tma_load_2d(st + 2 * a_bytes, &mapWhi, &full[slot], kcol, n0);
                        if (lo_too) tma_load_2d(st + 2 * a_bytes + b_bytes, &mapWlo, &full[slot], kcol, n0);
                        if (tr) { p.trace[p.trace_n + it] = clock64(); p.trace[9 * p.trace_n + it] = slot; }  // [1] loads issued, [9] slot
                        // k-block order: channel chunk outermost, taps inside
                        ++tap;
                        if (++kw == p.KW) { kw = 0; ++kh; }
                        if (tap == p.KH * p.KW) { tap = 0; kh = 0; kw = 0; c0 += kbc; }
                    }
                    if (p.trace && blockIdx.x == 0 && i < p.trace_n) p.trace[10 * p.trace_n + i] = skips;     // [10] held slot passed over
                }
            }
        }
    } else {
        if constexpr (epi_warps) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(TCP_REG_CONSUMER));
        // ================= consumer warpgroups: MMAs, chunk promotion, epilogue =================
        const int wg = warp >> 2;
        const uint32_t sbo = 8u * rowb, lay = rowb == 128u ? 2u : 4u;
        const int ksteps = (int)rowb / 32;
        const bool tr0 = p.trace && blockIdx.x == 0 && threadIdx.x == 0;
        int ph = 0, g = 0;                                      // ph bit s: parity of slot s's next fill
        int le = 0, lph = 0;                                    // slot_log entry of k-block g and the parity of its barrier
        auto acquire = [&]() {
            const bool tr = tr0 && g < p.trace_n;
            if (tr) p.trace[2 * p.trace_n + g] = clock64();                                    // [2] waiting for the stage
            mbar_wait(&log_bar[le], lph);
            // (a shuffle makes the slot warp-uniform for the compiler: read per thread, it costs the K loop ~20 registers and spills at BN = 128)
            const int s = __shfl_sync(0xffffffffu, slot_log[le], 0);
            if (++le > p.stages) { le = 0; lph ^= 1; }
            mbar_wait(&full[s], (ph >> s) & 1);
            ph ^= 1 << s;
            if (tr) p.trace[3 * p.trace_n + g] = clock64();                                    // [3] about to issue k-block g
            const uint32_t sa = smem_u32(smem + (size_t)s * stage_bytes);
            const uint32_t aw = sa + (uint32_t)wg * 64u * rowb;
            return KbOperands{make_sdesc(aw, sbo, lay), make_sdesc(aw + a_bytes, sbo, lay),
                              make_sdesc(sa + 2 * a_bytes, sbo, lay), make_sdesc(sa + 2 * a_bytes + b_bytes, sbo, lay), s};
        };
        auto release = [&](int st) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[st]);
        };
        auto issued = [&]() {
            if (tr0 && g < p.trace_n) p.trace[4 * p.trace_n + g] = clock64();                  // [4] k-block g issued, previous one retired
            ++g;
        };
        float tot[BN / 2], c[BN / 2];
        float amax = 0.f;                                       // (epilogue on the consumers)
        // the MMA mode and K steps per k-block are fixed per launch: one K loop per combination, chosen per tile outside the MMA chain
        auto kloop = [&](auto m, auto k) {
            return wg_tile_kloop<BN, F16, decltype(m)::value, decltype(k)::value>(tot, c, KB, p.chunk, acquire, release, issued, in_ring);
        };
        int i = 0;
        for (int u = u0; u < units; u += ustep, ++i) {
#pragma unroll
            for (int k = 0; k < BN / 2; ++k) tot[k] = 0.f;
            int held;                                           // (in_ring) slot of the tile's last k-block: the staging tile
            if (!F16 || ksteps == 4) {
                if (mode == 0) held = kloop(tc_int<0>(), tc_int<4>()); else if (mode == 2) held = kloop(tc_int<2>(), tc_int<4>()); else held = kloop(tc_int<1>(), tc_int<4>());
            } else {
                if (mode == 0) held = kloop(tc_int<0>(), tc_int<2>()); else if (mode == 2) held = kloop(tc_int<2>(), tc_int<2>()); else held = kloop(tc_int<1>(), tc_int<2>());
            }
            const bool tr = tr0 && i < p.trace_n;
            if (tr) p.trace[5 * p.trace_n + i] = clock64();                                     // [5] the tile's last MMAs are done
            float* tile = in_ring ? reinterpret_cast<float*>(smem + (size_t)held * stage_bytes) : tile_sep;
            if constexpr (!epi_warps) {
                // everyone is done reading the previous tile's staged accumulator, and (in_ring) both warpgroups' MMAs are done reading the held stage
                consumers_sync();
                wg_stage<BN>(tot, tile, LD, wg, warp, lane, swz);
                consumers_sync();
                bool pooled = false;
                if constexpr (BN == 64 && F16) {
                    if (p.pool_out) { tcp_pool_tile(p, tile, u, mt_units, warp, lane); pooled = true; }
                }
                if (!pooled) amax = fmaxf(amax, tcp_store_tile<BN>(p, tile, LD, u, mt_units, warp, lane, swz));
                if (in_ring) {
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // generic accesses to the stage before the next TMA write into it
                    release(held);
                }
            } else {
                // hand the tile to the epilogue warps and go on with the next one: the epilogue is done with the previous staged tile and the
                // mailbox (phase i - 1 of acc_empty; a fresh barrier passes parity 1), and (in_ring) both warpgroups' MMAs are done reading the held stage
                mbar_wait(acc_empty, (i & 1) ^ 1);
                consumers_sync();
                wg_stage<BN>(tot, split && wg == 1 ? tile_hi : tile, LD, wg, warp, lane, swz);
                if (threadIdx.x == 0) *mailbox = held;
                mbar_arrive(acc_full);
                if (tr) p.trace[6 * p.trace_n + i] = clock64();                                 // [6] staged and handed over
            }
        }
        note_fp16_range(amax, p.range_flag);
    }
}

// ----------------------------------------------------------------------------------------------------------------
// Gathered-row conv (vd3d_conv2d_tc16_gather): the M rows of a tile are 128 entries of a device list of output pixels, not a rectangle, and
// its N tile is one 96-column group of the output channels.  The anchor head's regression conv runs on the pixels whose anchors of that
// group the decoder reads (vd3d_reg_candidates), instead of on the whole map.
//   warps 0..7   two consumer warpgroups: the same wg_tile_kloop as conv2d_tcp_kernel (k-block order, chunk promotion, three products in
//                the same order), so every output element carries the bits the dense conv gives it (tile widths are bit-identical); the
//                epilogue (the dense one's arithmetic: scale, + 0 residual, + bias) stores straight from the accumulator registers, so no
//                staging tile takes shared memory from the operand ring
//   warp 8       weight producer: TMA boxes [64 k][96] of the (hi, lo) weight matrix, one per k-block
//   warps 9..12  gather: per k-block (tap, 64-channel chunk) 16-byte cp.async of every row's (hi, lo) channels into the SWIZZLE_128B K-major
//                stage (layout as dcn_fused.cu); a tap outside the image, a channel beyond Cin and a row beyond the list's count copy zero
//                bytes (zero fill), as the dense conv's TMA out-of-bounds fill does.  Each gather thread keeps TCG_LAG k-blocks of copies in
//                flight and signals a stage once its copies have landed.
// The tile count is read from the device (the list's per-group counts): the launch needs no host synchronisation.
// ----------------------------------------------------------------------------------------------------------------
constexpr int TCG_BN = 96;
constexpr int TCG_GATHER_WARPS = 4;
constexpr int TCG_THREADS = TC_CONSUMERS + 32 + 32 * TCG_GATHER_WARPS;
constexpr int TCG_STAGES = 4;
// k-blocks of copies a gather thread keeps in flight.  The consumers release a stage only after they have acquired the next one, so before
// the gather warps reuse the stage of k-block k - TCG_STAGES they must have signalled k-block k - TCG_STAGES + 1: TCG_LAG <= TCG_STAGES - 2.
constexpr int TCG_LAG = TCG_STAGES - 2;
constexpr int TCG_MAX_GROUPS = 32;

struct TcgParams {
    const __half* in_hi; const __half* in_lo;     // input planes [B][H][W][in_cs], channels in_co ..
    int H, W, in_cs, in_co;
    const int* list; const int* counts;           // list [groups][cap]: output pixel b * H * W + h * W + w; counts [groups]
    int groups, cap;
    int KW, taps, pad, dil;
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}

__global__ void __launch_bounds__(TCG_THREADS, 1)
conv2d_tcg_kernel(const __grid_constant__ CUtensorMap mapWhi, const __grid_constant__ CUtensorMap mapWlo, const TcParams p, const TcgParams g) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    constexpr int BN = TCG_BN;
    constexpr uint32_t a_bytes = 128u * 128u, b_bytes = (uint32_t)BN * 128u, stage_bytes = 2u * a_bytes + 2u * b_bytes;
    uint64_t* fullA = reinterpret_cast<uint64_t*>(smem + (size_t)TCG_STAGES * stage_bytes);   // [stages] gather warps -> consumers
    uint64_t* fullB = fullA + TCG_STAGES;                                                 // [stages] weight TMA -> consumers
    uint64_t* empty = fullB + TCG_STAGES;                                                 // [stages] consumers (8 warps) -> producers
    int* first = reinterpret_cast<int*>(empty + TCG_STAGES);                              // [groups + 1] first tile of each group

    const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
    const int KB = g.taps * (p.cin_pad / 64);
    if (threadIdx.x == 0) {
        for (int s = 0; s < TCG_STAGES; ++s) { mbar_init(&fullA[s], TCG_GATHER_WARPS); mbar_init(&fullB[s], 1); mbar_init(&empty[s], TC_CONSUMERS / 32); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    pdl_launch_dependents();
    pdl_wait();                            // (PDL launches only) the list and the input planes are complete
    if (threadIdx.x == 0) {
        int t = 0;
        for (int q = 0; q < g.groups; ++q) { first[q] = t; t += (__ldg(g.counts + q) + 127) / 128; }
        first[g.groups] = t;
    }
    __syncthreads();
    const int units = first[g.groups];
    // tile u -> group, its first list entry and the number of entries of the group
    auto tile_of = [&](int u, int& grp, int& e0, int& cnt) {
        grp = 0;
        while (u >= first[grp + 1]) ++grp;
        e0 = (u - first[grp]) * 128;
        cnt = __ldg(g.counts + grp);
    };
    // k-block kb = (64-channel chunk, tap), chunk outermost: the K order of conv2d_tcp_kernel
    auto kcol = [&](int kb, int& tap, int& c0) { tap = kb % g.taps; c0 = (kb / g.taps) * 64; };

    if (warp == TC_CONSUMERS / 32) {
        // ================= weight producer =================
        int it = 0;
        for (int u = (int)blockIdx.x; u < units; u += (int)gridDim.x) {
            int grp, e0, cnt;
            tile_of(u, grp, e0, cnt);
            for (int kb = 0; kb < KB; ++kb, ++it) {
                const int s = it % TCG_STAGES, ph = (it / TCG_STAGES) & 1;
                mbar_wait(&empty[s], ph ^ 1);
                if (elect_one()) {
                    int tap, c0;
                    kcol(kb, tap, c0);
                    uint8_t* st = smem + (size_t)s * stage_bytes + 2 * a_bytes;
                    mbar_expect_tx(&fullB[s], 2u * b_bytes);
                    tma_load_2d(st, &mapWhi, &fullB[s], tap * p.cin_pad + c0, grp * BN);
                    tma_load_2d(st + b_bytes, &mapWlo, &fullB[s], tap * p.cin_pad + c0, grp * BN);
                }
                __syncwarp();
            }
        }
    } else if (warp < TC_CONSUMERS / 32) {
        // ================= consumer warpgroups =================
        const int wg = warp >> 2;
        int it = 0;
        auto acquire = [&]() {
            const int s = it % TCG_STAGES, ph = (it / TCG_STAGES) & 1;
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
        // accumulator fragment (wg_stage): rows 64 wg + 16 (warp % 4) + lane / 4 (+ 8), columns 8 i + 2 (lane % 4) (+ 1)
        const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
        for (int u = (int)blockIdx.x; u < units; u += (int)gridDim.x) {
            int grp, e0, cnt;
            tile_of(u, grp, e0, cnt);
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) tot[i] = 0.f;
            wg_tile_kloop<BN, true, 0, 4>(tot, c, KB, p.chunk, acquire, release, issued);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (e0 + r0 + 8 * h >= cnt) continue;
                const long long pix = __ldg(g.list + (long long)grp * g.cap + e0 + r0 + 8 * h);
                float* op = p.out + pix * p.out_cs + p.out_co;
#pragma unroll
                for (int i = 0; i < BN / 8; ++i) {
                    const int n = grp * BN + 8 * i + c0;
                    if (n < p.Cout) {                             // (n even, Cout % 4 == 0: both columns exist)
                        const float2 bb = p.bias ? __ldg(reinterpret_cast<const float2*>(p.bias + n)) : make_float2(0.f, 0.f);
                        float a0 = tot[4 * i + 2 * h] * p.out_scale + 0.f, a1 = tot[4 * i + 2 * h + 1] * p.out_scale + 0.f;   // tcp_epi_out, no residual
                        a0 += bb.x; a1 += bb.y;
                        *reinterpret_cast<float2*>(op + n) = make_float2(a0, a1);
                    }
                }
            }
        }
    } else {
        // ================= gather warps =================
        const int gt = (int)threadIdx.x - (TC_CONSUMERS + 32);
        const int j = gt & 7;                                  // 16-byte chunk (8 channels) of the 64-channel k-block
        const int m0 = gt >> 3;                                // rows m0 + 16 r, r = 0 .. 7
        constexpr int ROWS = 128 / (TCG_GATHER_WARPS * 4);
        const int HW = g.H * g.W;
        int it = 0;
        auto signal = [&](int k) {                             // the copies of k-block k (and every earlier one) have landed
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic-proxy writes -> the tensor core's async-proxy reads
            __syncwarp();
            if (lane == 0) mbar_arrive(&fullA[k % TCG_STAGES]);
        };
        for (int u = (int)blockIdx.x; u < units; u += (int)gridDim.x) {
            int grp, e0, cnt;
            tile_of(u, grp, e0, cnt);
            int pix[ROWS], ph_[ROWS], pw_[ROWS];               // output pixel of each row (-1: beyond the count), its row / column
#pragma unroll
            for (int r = 0; r < ROWS; ++r) {
                const int e = e0 + m0 + 16 * r;
                pix[r] = e < cnt ? __ldg(g.list + (long long)grp * g.cap + e) : -1;
                const int pi = pix[r] < 0 ? 0 : pix[r] % HW;
                ph_[r] = pi / g.W; pw_[r] = pi - ph_[r] * g.W;
            }
            for (int kb = 0; kb < KB; ++kb, ++it) {
                const int s = it % TCG_STAGES, ph = (it / TCG_STAGES) & 1;
                mbar_wait(&empty[s], ph ^ 1);
                int tap, c0;
                kcol(kb, tap, c0);
                const int kh = tap / g.KW, kw = tap - kh * g.KW;
                const int dy = kh * g.dil - g.pad, dx = kw * g.dil - g.pad;
                const int ch = c0 + 8 * j;
                const uint32_t sa = smem_u32(smem + (size_t)s * stage_bytes);
#pragma unroll
                for (int r = 0; r < ROWS; ++r) {
                    const int m = m0 + 16 * r;
                    const int hi = ph_[r] + dy, wi = pw_[r] + dx;
                    const bool ok = pix[r] >= 0 && (unsigned)hi < (unsigned)g.H && (unsigned)wi < (unsigned)g.W && ch < p.Cin;
                    const long long off = ok ? (long long)(pix[r] + dy * g.W + dx) * g.in_cs + g.in_co + ch : 0;
                    const uint32_t so = (uint32_t)(m >> 3) * 1024u + (uint32_t)(m & 7) * 128u + (uint32_t)((j ^ (m & 7)) * 16);
                    cp_async16(sa + so, g.in_hi + off, ok ? 16u : 0u);
                    cp_async16(sa + a_bytes + so, g.in_lo + off, ok ? 16u : 0u);
                }
                asm volatile("cp.async.commit_group;" ::: "memory");
                if (it >= TCG_LAG) {
                    asm volatile("cp.async.wait_group %0;" ::"n"(TCG_LAG) : "memory");
                    signal(it - TCG_LAG);
                }
            }
        }
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        for (int k = it - TCG_LAG < 0 ? 0 : it - TCG_LAG; k < it; ++k) signal(k);
    }
}

// lo = v - (v & 0xFFFFE000): the part of v the tf32 MMA does not see.  Elementwise, float4, channel-slice aware.
__global__ void split_lo_kernel(const float* __restrict__ in, float* __restrict__ lo, long long npix, int C4, int cs, int co) {
    long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= npix * C4) return;
    int c4 = (int)(idx % C4); long long pix = idx / C4;
    float4 a = ldg4(in + pix * cs + co + 4 * c4);
    float4 l;
    l.x = a.x - __uint_as_float(__float_as_uint(a.x) & 0xFFFFE000u);
    l.y = a.y - __uint_as_float(__float_as_uint(a.y) & 0xFFFFE000u);
    l.z = a.z - __uint_as_float(__float_as_uint(a.z) & 0xFFFFE000u);
    l.w = a.w - __uint_as_float(__float_as_uint(a.w) & 0xFFFFE000u);
    *reinterpret_cast<float4*>(lo + pix * cs + co + 4 * c4) = l;
}

// fp32 -> fp16 (hi, lo) planes: hi = rn16(v), lo = rn16(v - hi).  Elementwise, channel-slice aware (planes share the fp32 pitch).
__global__ void split_h16_kernel(const float* __restrict__ in, __half* __restrict__ hi, __half* __restrict__ lo, long long npix, int C4, int cs, int co,
                                 int* __restrict__ range_flag) {
    long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= npix * C4) return;
    int c4 = (int)(idx % C4); long long pix = idx / C4;
    float4 a = ldg4(in + pix * cs + co + 4 * c4);
    note_fp16_range(amax4(0.f, a), range_flag);
    __half hx = __float2half_rn(a.x), hy = __float2half_rn(a.y), hz = __float2half_rn(a.z), hw = __float2half_rn(a.w);
    __half2 h01 = __halves2half2(hx, hy), h23 = __halves2half2(hz, hw);
    __half2 l01 = __halves2half2(__float2half_rn(a.x - __half2float(hx)), __float2half_rn(a.y - __half2float(hy)));
    __half2 l23 = __halves2half2(__float2half_rn(a.z - __half2float(hz)), __float2half_rn(a.w - __half2float(hw)));
    uint2 hv, lv;
    hv.x = *reinterpret_cast<uint32_t*>(&h01); hv.y = *reinterpret_cast<uint32_t*>(&h23);
    lv.x = *reinterpret_cast<uint32_t*>(&l01); lv.y = *reinterpret_cast<uint32_t*>(&l23);
    *reinterpret_cast<uint2*>(hi + pix * cs + co + 4 * c4) = hv;
    *reinterpret_cast<uint2*>(lo + pix * cs + co + 4 * c4) = lv;
}

// ----------------------------------------------------------------------------------------------------------------
// host: tensor maps (driver entry point fetched at run time: the library does not link libcuda)
// ----------------------------------------------------------------------------------------------------------------
// `stride` > 1: TMA traversal stride (elementStrides) on W and H, so the box holds every stride-th pixel: a strided conv
// reads exactly the 16 x 8 input pixels its 128 outputs need for one tap, densely packed in shared memory.
static int make_map_act(CUtensorMap* m, const void* base_v, int B, int H, int W, int C, int cs, int co, int esize = 4,
                        int box_w = TC_TW, int box_h = TC_TH, int stride = 1) {
    EncodeTiledFn enc = get_encode();
    if (!enc) { set_error("conv2d_tc: cuTensorMapEncodeTiled unavailable"); return VD3D_ECUDA; }
    const char* base = (const char*)base_v + (size_t)co * esize;
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)cs * esize, (cuuint64_t)W * cs * esize, (cuuint64_t)H * W * cs * esize};
    cuuint32_t box[4] = {(cuuint32_t)(128 / esize), (cuuint32_t)(box_w * stride), (cuuint32_t)(box_h * stride), 1};
    cuuint32_t es[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
    CUresult r = enc(m, esize == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, (void*)base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("conv2d_tc: cuTensorMapEncodeTiled(activation) failed: %d", (int)r); return VD3D_ECUDA; }
    return VD3D_OK;
}

}  // namespace vd3d

using namespace vd3d;

// persistent fp16 engine: the widest tile (<= TC_MAX_BN) that splits Cout evenly into ceil(Cout / TC_MAX_BN) tiles of 16-column granules
extern "C" int vd3d_tc_pick_bn_persistent(int Cout) {
    const int cp = (Cout + 15) / 16 * 16;
    const int nt = (cp + TC_MAX_BN - 1) / TC_MAX_BN;
    return ((cp + nt - 1) / nt + 15) / 16 * 16;
}

// Tile width for a given problem: minimise  rounds x (BN + 64)  over 16-column granules, where rounds = ceil(tiles / SMs) and the
// constant stands for the per-k-block cost that does not scale with the tile width (barrier / issue gaps and the epilogue).
static int pick_bn_cost(int Cout, int m_tiles) {
    const int cp = (Cout + 15) / 16 * 16;
    if (cp <= TC_MAX_BN) return cp;
    int best = vd3d_tc_pick_bn_persistent(Cout);
    long long best_cost = -1;
    for (int bn = 64; bn <= TC_MAX_BN; bn += 16) {
        const long long units = (long long)m_tiles * ((cp + bn - 1) / bn);
        const long long rounds = (units + kNumSMs - 1) / kNumSMs;
        const long long cost = rounds * (bn + 64);
        if (best_cost < 0 || cost < best_cost || (cost == best_cost && bn > best)) { best_cost = cost; best = bn; }
    }
    return best;
}

extern "C" int vd3d_tc_pick_bn(int Cout) {
    // largest tile <= 128 that divides Cout evenly into 16-multiples; otherwise the single-tile / 64 fallbacks
    if (Cout % 128 == 0) return 128;
    if (Cout < 128 && Cout % 16) return (Cout + 15) / 16 * 16;        // single N tile, columns >= Cout masked (weight rows beyond Cout are TMA zero fill)
    if (Cout % 96 == 0) return 96;
    if (Cout % 64 == 0) return 64;
    if (Cout % 48 == 0) return 48;
    if (Cout % 32 == 0) return 32;
    return Cout <= 128 ? (Cout + 15) / 16 * 16 : 128;
}

// diagnostics: clock64 stamps of the TMA / MMA pipeline and the tile hand-off of CTA 0 ([12][n] int64 device buffer; NULL disables)
static long long* g_trace = nullptr;
static int g_trace_n = 0;
extern "C" void vd3d_tc_set_trace(void* dev_i64, int n) { g_trace = (long long*)dev_i64; g_trace_n = n; }

// launch of the persistent kernel: p.BN (<= TC_MAX_BN) / p.chunk / tile counts are set by the caller, the weight maps have BN rows per box;
// `lm`: the per-level activation maps of a multi-level launch (p.n_levels > 0, fp16 operands only)
static int tcp_launch(TcParams& p, const CUtensorMap& mA, const CUtensorMap& mAlo, const CUtensorMap& mWhi, const CUtensorMap& mWlo, void* stream,
                      const TcLevelMaps* lm = nullptr) {
    const int BN = p.BN;
    { const char* e = getenv("VD3D_TC_DEBUG"); p.dbg = e ? atoi(e) : 0; }
    p.trace = g_trace; p.trace_n = g_trace_n;
    if (p.rowb == 0) p.rowb = 128;
    VD3D_REQUIRE(BN % 16 == 0 && BN >= 16 && BN <= TC_MAX_BN, "conv2d_tc: BN must be a multiple of 16 in [16, %d]", TC_MAX_BN);
    const size_t stage_bytes = 2 * (size_t)128 * p.rowb + 2 * (size_t)BN * p.rowb;
    VD3D_REQUIRE(!p.pool_out || (BN == 64 && p.f16 && p.relu && !p.res && !p.res_h16_hi), "conv2d_tc: the fused max-pool needs a 64-column fp16 tile with ReLU and no residual");
    // Staging tile: a separate tile after the ring, or the stage of the tile's last k-block (which then stays held through the epilogue) when
    // the accumulator fits there and that buys a stage; the producer still gets as many stages for the next tile while the epilogue runs as
    // with a separate tile.  VD3D_TC_TILE_IN_RING=0 always uses a separate tile.
    const size_t avail = 227 * 1024 - 1024 - 256;
    const size_t tile_bytes = (size_t)128 * tcp_tile_ld(BN) * sizeof(float);
    int stages = (int)((avail - tile_bytes) / stage_bytes);
    {
        const char* e = getenv("VD3D_TC_TILE_IN_RING");
        const int stages_in = (int)(avail / stage_bytes);
        p.tile_in_ring = !(e && atoi(e) == 0) && tile_bytes <= stage_bytes && stages < 8 && stages_in > stages;
        if (p.tile_in_ring) stages = stages_in;
    }
    if (stages > 8) stages = 8;
    VD3D_REQUIRE(stages >= 2, "conv2d_tc: tile too large for shared memory");
    p.stages = stages;
    // Split staging (epilogue warps only): when half a staging tile fits next to the ring, rows 64..127 of the accumulator go there and the
    // held stage is released halfway through the epilogue.  Never at the cost of a stage.
    const size_t half_bytes = tile_bytes / 2;
    p.split_stage = p.tile_in_ring && tcp_epi_warps(BN) && stages * stage_bytes + half_bytes <= avail;
    // barrier area: full[stages], empty[stages], log_bar[stages + 1], acc_full, acc_empty; then the mailbox and slot_log[stages + 1]
    // (at most 256 bytes: 8 stages)
    const size_t bar_bytes = ((3 * stages + 3) * sizeof(uint64_t) + (stages + 2) * sizeof(int) + 15) / 16 * 16;
    const size_t smem = stages * stage_bytes + (p.tile_in_ring ? (p.split_stage ? half_bytes : 0) : tile_bytes) + bar_bytes + 1024;
    const int units = p.m_tiles * p.n_tiles;
    int grid = units < kNumSMs ? units : kNumSMs;
    { const char* e = getenv("VD3D_TC_GRID"); const int cap = e ? atoi(e) : 0; if (cap > 0 && cap < grid) grid = cap; }     // diagnostics
    cudaError_t le = cudaErrorInvalidValue;
    VD3D_REQUIRE(!lm || (p.f16 && p.n_levels > 0), "conv2d_tc: multi-level launches take fp16 operands");
    const TcNoLevelMaps nolm{0};
#define VD3D_TCP_LAUNCH(N, F16, LV, LM) tc_launch<conv2d_tcp_kernel<N, F16, LV>>(grid, tcp_threads(N), smem, stream, mA, mAlo, mWhi, mWlo, p, LM)
#define VD3D_TCP_CASE(N) case N: le = lm ? VD3D_TCP_LAUNCH(N, true, true, *lm) : p.f16 ? VD3D_TCP_LAUNCH(N, true, false, nolm) : VD3D_TCP_LAUNCH(N, false, false, nolm); break
    switch (BN) {
        VD3D_TCP_CASE(16); VD3D_TCP_CASE(32); VD3D_TCP_CASE(48); VD3D_TCP_CASE(64);
        VD3D_TCP_CASE(80); VD3D_TCP_CASE(96); VD3D_TCP_CASE(112); VD3D_TCP_CASE(128);
    }
#undef VD3D_TCP_CASE
#undef VD3D_TCP_LAUNCH
    if (le != cudaSuccess) { set_error("conv2d_tcp: launch failed: %s", cudaGetErrorString(le)); return VD3D_ECUDA; }
    VD3D_CHECK_LAUNCH("conv2d_tcp");
    return VD3D_OK;
}

// a requested tile wider than TC_MAX_BN runs as equal halves (16-column granules): every width accumulates identically
static int fit_bn(int bn) {
    while (bn > TC_MAX_BN) bn = (bn / 2 + 15) / 16 * 16;
    return bn;
}

// One conv as the entries describe it: L input tensors of one channel layout (L > 1: a multi-level launch, fp16 operands only), the weights
// and the epilogue.  Level l reads in[l] / in_lo[l] [B][H[l]][W[l]]; its outputs and fp32 residual lie out_off[l] / res_off[l] pixels after
// level 0's (L > 1); res_W[l] > 0: its fp32 residual is [B][res_H[l]][res_W[l]] at half the output size, read nearest-upsampled.
// convt: the four sub-pixel phases of a 4x4 / stride-2 / pad-1 transposed conv (vd3d_convtranspose2d_tc16): L = 4 levels over one input,
// 2x2 taps each, weights [4 Cout][4 cin_pad] (phase l = 2 r + s owns rows l Cout ..), output [B][2 H][2 W].
struct ConvSpec {
    int f16, L, B, Cin, in_cs, in_co;
    const void* in[TC_MAX_LEVELS]; const void* in_lo[TC_MAX_LEVELS];
    int H[TC_MAX_LEVELS], W[TC_MAX_LEVELS], res_H[TC_MAX_LEVELS], res_W[TC_MAX_LEVELS];
    long long out_off[TC_MAX_LEVELS], res_off[TC_MAX_LEVELS];
    const void* w_hi; const void* w_lo; float out_scale; const float* bias;
    int KH, KW, pad, dil, stride;
    const float* res; const void* res_h16_hi; const void* res_h16_lo; int res_cs, res_co;
    float* out; float* out_lo; void* out_h16_hi; void* out_h16_lo;
    int Cout, out_cs, out_co, relu, passes, bn;
    int convt;
    const int4* tlist; const int* tcount; const uint8_t* smap;     // tile-listed launch (TcParams::tlist)
};

// output size of level l: the conv's, or (convt) the input's -- each phase writes one pixel of every 2x2 output cell
static void spec_out_hw(const ConvSpec& s, int l, int& Ho, int& Wo) {
    if (s.convt) { Ho = s.H[l]; Wo = s.W[l]; return; }
    Ho = (s.H[l] + 2 * s.pad - s.dil * (s.KH - 1) - 1) / s.stride + 1;
    Wo = (s.W[l] + 2 * s.pad - s.dil * (s.KW - 1) - 1) / s.stride + 1;
}

static int conv2d_tc_launch(const ConvSpec& s, void* stream) {
    const int f16 = s.f16, B = s.B, H = s.H[0], W = s.W[0], Cin = s.Cin, KH = s.KH, KW = s.KW, pad = s.pad, dil = s.dil, stride = s.stride;
    const int Cout = s.Cout, out_cs = s.out_cs, out_co = s.out_co, res_cs = s.res_cs, res_co = s.res_co;
    VD3D_REQUIRE(s.in[0] && s.w_hi && (s.out || s.out_h16_hi), "conv2d_tc: null pointer");
    VD3D_REQUIRE(!(s.res && s.res_h16_hi) && (!s.res_h16_hi == !s.res_h16_lo), "conv2d_tc: the residual is either an fp32 tensor or an fp16 (hi, lo) plane pair");
    int passes = s.passes;
    const int two_pass = (f16 && passes == 2) ? 1 : 0;        // error-budget experiments: 3-pass machinery with the A_lo * W_hi product dropped
    if (two_pass) passes = 3;
    VD3D_REQUIRE(passes == 1 || passes == 3, "conv2d_tc: passes must be 1, 3 (or 2 with the fp16-split engine)");
    VD3D_REQUIRE(passes == 1 || (s.in_lo[0] && s.w_lo), "conv2d_tc: 3-pass mode needs the lo tensors");
    VD3D_REQUIRE(!(two_pass && s.res_h16_hi), "conv2d_tc: the 2-pass experiment takes an fp32 residual only");
    const int esize = f16 ? 2 : 4, bk = 128 / esize;
    VD3D_REQUIRE(f16 ? (Cin % 8 == 0) : (Cin % bk == 0), "conv2d_tc: Cin must be a multiple of %d (got %d)", f16 ? 8 : bk, Cin);
    VD3D_REQUIRE(s.in_cs % 8 == 0 && s.in_co % 8 == 0 && out_cs % 4 == 0 && out_co % 4 == 0 && Cout % 4 == 0, "conv2d_tc: pitches/offsets alignment");
    VD3D_REQUIRE(!(s.res || s.res_h16_hi) || (res_cs % 4 == 0 && res_co % 4 == 0), "conv2d_tc: residual pitch/offset must be multiples of 4");
    VD3D_REQUIRE(((uintptr_t)s.in[0] & 15) == 0 && ((uintptr_t)s.w_hi & 15) == 0 && ((uintptr_t)s.out & 15) == 0, "conv2d_tc: pointers must be 16-byte aligned");
    VD3D_REQUIRE(!s.res_h16_hi || ((((uintptr_t)s.res_h16_hi | (uintptr_t)s.res_h16_lo) & 7) == 0), "conv2d_tc: residual planes must be 8-byte aligned");
    VD3D_REQUIRE(!s.out_h16_hi || (s.out_h16_lo && out_cs % 4 == 0), "conv2d_tc: fp16 output planes come in (hi, lo) pairs");
    int BN = s.bn;
    if (BN <= 0) {
        if (f16 && passes == 3) {
            int mt_all = 0;
            for (int l = 0; l < s.L; ++l) {
                int Ho_, Wo_;
                spec_out_hw(s, l, Ho_, Wo_);
                mt_all += cdiv(Wo_, TC_TW) * cdiv(Ho_, TC_TH) * B;
            }
            BN = pick_bn_cost(Cout, mt_all);
        } else BN = vd3d_tc_pick_bn(Cout);
    }
    VD3D_REQUIRE(BN % 16 == 0 && BN >= 16 && BN <= 256, "conv2d_tc: BN must be a multiple of 16 in [16, 256]");
    BN = fit_bn(BN);
    TcParams p;
    memset(&p, 0, sizeof(p));
    VD3D_REQUIRE(stride >= 1 && stride <= 4, "conv2d_tc: stride must be in [1, 4]");
    p.B = B; p.H = H; p.W = W; p.Cin = Cin; p.KH = KH; p.KW = KW; p.pad = pad; p.dil = dil; p.stride = stride;
    spec_out_hw(s, 0, p.Ho, p.Wo);
    VD3D_REQUIRE(p.Ho > 0 && p.Wo > 0, "conv2d_tc: empty output");
    p.Cout = Cout; p.BN = BN; p.passes = passes; p.f16 = f16; p.bk = bk; p.cin_pad = (Cin + bk - 1) / bk * bk; p.out_scale = s.out_scale;
    p.tiles_w = cdiv(p.Wo, TC_TW); p.tiles_h = cdiv(p.Ho, TC_TH);
    p.stride_w = stride; p.pad_w = pad;
    p.cout_pad = (Cout + 15) / 16 * 16;
    p.m_tiles = p.tiles_w * p.tiles_h * B; p.n_tiles = cdiv(p.cout_pad, BN);
    p.rowb = 128;
    if (s.L > 1) {
        // concatenated M tiles of the levels (tile_geom); the level's own maps give each its zero padding
        VD3D_REQUIRE(s.L <= TC_MAX_LEVELS && f16 && s.passes == 3 && !s.res_h16_hi, "conv2d_tc16: bad level set");
        p.n_levels = s.L;
        int mt = 0;
        for (int l = 0; l < s.L; ++l) {
            TcLevel& v = p.lv[l];
            spec_out_hw(s, l, v.Ho, v.Wo);
            VD3D_REQUIRE(v.Ho > 0 && v.Wo > 0, "conv2d_tc16: level %d has an empty output", l);
            v.pad_h = pad; v.pad_w = pad; v.w_row = 0; v.up = 0;
            if (s.convt) {
                // phase (r, s) = (l >> 1, l & 1): y[2m + r][2n + s] = sum_{a,b} x[m + r - 1 + a][n + s - 1 + b] W_rs[a][b]
                const int r = l >> 1, c = l & 1;
                v.pad_h = 1 - r; v.pad_w = 1 - c; v.w_row = l * Cout; v.up = 1;
            }
            v.tiles_w = cdiv(v.Wo, TC_TW); v.tiles_h = cdiv(v.Ho, TC_TH);
            v.m_begin = mt;
            mt += v.tiles_w * v.tiles_h * B;
            v.pix_off = s.out_off[l]; v.res_off = s.res_off[l];
            v.res_H = s.res_H[l]; v.res_W = s.res_W[l];
            VD3D_REQUIRE(v.res_W == 0 || (s.res && v.Ho == 2 * v.res_H && v.Wo == 2 * v.res_W),
                         "conv2d_tc16: level %d: an upsampled residual needs exactly half the output size", l);
        }
        p.m_tiles = mt;
    }
    {
        // L2-aware tile order (unit_tile): M blocks whose activation slab (the block's input pixels, all channels, both planes) is about
        // VD3D_TC_L2MB megabytes (default 20: well inside the 50 MB L2), only when there is more than one N tile (otherwise A is read once
        // anyway).  0 disables.
        const char* e = getenv("VD3D_TC_L2MB");
        const double l2mb = e ? atof(e) : 20.0;
        p.mblock = 0;
        if (p.n_tiles > 1 && l2mb > 0) {
            const double a_bytes_per_tile = 128.0 * stride * stride * (double)p.cin_pad * (f16 ? 4.0 : 8.0);
            int mb = (int)(l2mb * 1048576.0 / a_bytes_per_tile);
            if (mb < 8) mb = 8;
            if (mb < p.m_tiles) {
                const int nblk = cdiv(p.m_tiles, mb);
                p.mblock = cdiv(p.m_tiles, nblk);       // equal blocks
            }
        }
    }
    p.v8 = (out_cs % 8 == 0 && out_co % 8 == 0 && ((uintptr_t)s.out & 31) == 0 && (!s.bias || ((uintptr_t)s.bias & 31) == 0) &&
            (!s.res || (res_cs % 8 == 0 && res_co % 8 == 0 && ((uintptr_t)s.res & 31) == 0)) &&
            (!s.res_h16_hi || (res_cs % 8 == 0 && res_co % 8 == 0 && ((((uintptr_t)s.res_h16_hi | (uintptr_t)s.res_h16_lo) & 15) == 0))) &&
            (!s.out_h16_hi || ((((uintptr_t)s.out_h16_hi | (uintptr_t)s.out_h16_lo) & 15) == 0))) ? 1 : 0;
    p.out_cs = out_cs; p.out_co = out_co; p.res_cs = res_cs; p.res_co = res_co; p.relu = s.relu;
    p.bias = s.bias; p.res = s.res; p.out = s.out; p.out_lo = s.out_lo; p.out_h16_hi = s.out_h16_hi; p.out_h16_lo = s.out_h16_lo;
    p.res_h16_hi = s.res_h16_hi; p.res_h16_lo = s.res_h16_lo;
    if (s.L == 1 && s.res_W[0] > 0) {
        const int res_up_H = s.res_H[0], res_up_W = s.res_W[0];
        VD3D_REQUIRE(s.res && !s.res_h16_hi && p.Ho == 2 * res_up_H && p.Wo == 2 * res_up_W,
                     "conv2d_tc: an upsampled residual is an fp32 tensor of exactly half the output size (%dx%d vs %dx%d)", res_up_H, res_up_W, p.Ho, p.Wo);
        p.res_up_H = res_up_H; p.res_up_W = res_up_W;
    }
    p.two_pass = two_pass;
    if (s.tlist) {
        // the list's origins are output pixels of a stride-1 conv over one tensor; the fused pool writes whole pooled tiles
        VD3D_REQUIRE(s.L == 1 && stride == 1 && f16 && passes == 3 && !two_pass && !s.convt && s.res_W[0] == 0 && s.tcount && s.smap,
                     "conv2d_tc16_tiles: a tile list needs a one-tensor, stride-1 fp16-split conv, its device count and a store map");
        p.tlist = s.tlist; p.tcount = s.tcount; p.smap = s.smap;
    }
    p.range_flag = s.out_h16_hi ? fp16_range_flag() : nullptr;
    {
        const char* e = getenv("VD3D_TC_CHUNK");
        p.chunk = e ? atoi(e) : 4;
        if (p.chunk < 1) p.chunk = 1;
    }
    {
        // 64-channel 3x3 convs: the row-strip kernel (conv2d_row64.cu, same bits).  VD3D_ROW64=0 keeps them on conv2d_tcp_kernel, as do the
        // MMA-mode timing experiments (VD3D_TC_DEBUG bits 0 and 1), which only conv2d_tcp_kernel implements.
        const char* e = getenv("VD3D_ROW64");
        const char* d = getenv("VD3D_TC_DEBUG");
        if (s.L == 1 && !s.tlist && conv2d_row64_eligible(p) && !(e && atoi(e) == 0) && !(d && (atoi(d) & 3)))
            return conv2d_row64_launch(p, s.in[0], s.in_lo[0], s.in_cs, s.in_co, s.w_hi, s.w_lo, stream);
    }
    const int K = KH * KW * p.cin_pad;
    CUtensorMap mA, mAlo, mWhi, mWlo;
    int rc;
    if ((rc = make_map_act(&mA, s.in[0], B, H, W, Cin, s.in_cs, s.in_co, esize, TC_TW, TC_TH, stride))) return rc;
    if ((rc = make_map_act(&mAlo, s.in_lo[0] ? s.in_lo[0] : s.in[0], B, H, W, Cin, s.in_cs, s.in_co, esize, TC_TW, TC_TH, stride))) return rc;
    const int w_rows = s.convt ? 4 * Cout : Cout;
    if ((rc = make_map_wgt(&mWhi, s.w_hi, w_rows, K, BN, esize))) return rc;
    if ((rc = make_map_wgt(&mWlo, s.w_lo ? s.w_lo : s.w_hi, w_rows, K, BN, esize))) return rc;
    if (s.L == 1) return tcp_launch(p, mA, mAlo, mWhi, mWlo, stream);
    TcLevelMaps lm;
    for (int l = 0; l < s.L; ++l) {
        if ((rc = make_map_act(&lm.a[l], s.in[l], B, s.H[l], s.W[l], Cin, s.in_cs, s.in_co, esize, TC_TW, TC_TH, stride))) return rc;
        if ((rc = make_map_act(&lm.alo[l], s.in_lo[l], B, s.H[l], s.W[l], Cin, s.in_cs, s.in_co, esize, TC_TW, TC_TH, stride))) return rc;
    }
    return tcp_launch(p, mA, mAlo, mWhi, mWlo, stream, &lm);
}

// pixel offset of level l's tensor relative to level 0's, from the two base pointers (bytes / (esize * cs)); -1 LL << 62 if not a whole pixel
static long long level_pix_off(const void* base0, const void* base, int esize, int cs) {
    const long long d = (long long)((const char*)base - (const char*)base0);
    return d % ((long long)esize * cs) ? (-1LL << 62) : d / ((long long)esize * cs);
}

extern "C" int vd3d_conv2d_tc(const float* in, const float* in_lo, int B, int H, int W, int Cin, int in_cs, int in_co,
                              const float* w_hi, const float* w_lo, const float* bias, int KH, int KW, int pad, int dil,
                              const float* res, int res_cs, int res_co,
                              float* out, float* out_lo, int Cout, int out_cs, int out_co, int relu, int passes, int bn, void* stream) {
    ConvSpec s;
    memset(&s, 0, sizeof(s));
    s.f16 = 0; s.L = 1; s.B = B; s.Cin = Cin; s.in_cs = in_cs; s.in_co = in_co;
    s.in[0] = in; s.in_lo[0] = in_lo; s.H[0] = H; s.W[0] = W;
    s.w_hi = w_hi; s.w_lo = w_lo; s.out_scale = 1.0f; s.bias = bias;
    s.KH = KH; s.KW = KW; s.pad = pad; s.dil = dil; s.stride = 1;
    s.res = res; s.res_cs = res_cs; s.res_co = res_co;
    s.out = out; s.out_lo = out_lo;
    s.Cout = Cout; s.out_cs = out_cs; s.out_co = out_co; s.relu = relu; s.passes = passes; s.bn = bn;
    return conv2d_tc_launch(s, stream);
}

extern "C" int vd3d_conv2d_tc16(int L, const void* const* in_hi, const void* const* in_lo, const int* H, const int* W, int B, int Cin, int in_cs,
                                int in_co, const void* w_hi, const void* w_lo, float out_scale, const float* bias, int KH, int KW, int pad,
                                int dil, int stride, const void* const* res, const void* const* res_hi16, const void* const* res_lo16,
                                const int* res_H, const int* res_W, int res_cs, int res_co,
                                const void* const* out, const void* const* out_hi16, const void* const* out_lo16,
                                int Cout, int out_cs, int out_co, int relu, int passes, int bn, void* stream) {
    VD3D_REQUIRE(L >= 1 && L <= TC_MAX_LEVELS && in_hi && in_lo && H && W && (out || out_hi16) && (!out_hi16 == !out_lo16) &&
                 (!res_hi16 == !res_lo16), "conv2d_tc16: 1..%d levels, inputs, sizes and an output are required", TC_MAX_LEVELS);
    ConvSpec s;
    memset(&s, 0, sizeof(s));
    s.f16 = 1; s.L = L; s.B = B; s.Cin = Cin; s.in_cs = in_cs; s.in_co = in_co;
    for (int l = 0; l < L; ++l) {
        VD3D_REQUIRE(in_hi[l] && in_lo[l] && H[l] > 0 && W[l] > 0 && ((((uintptr_t)in_hi[l] | (uintptr_t)in_lo[l]) & 15) == 0),
                     "conv2d_tc16: level %d: 16-byte aligned input planes and a non-empty size are required", l);
        s.in[l] = in_hi[l]; s.in_lo[l] = in_lo[l]; s.H[l] = H[l]; s.W[l] = W[l];
        s.res_H[l] = res_H ? res_H[l] : 0; s.res_W[l] = res_W ? res_W[l] : 0;
        // every output form of level l sits at the same pixel offset from level 0's (one allocation per form, levels concatenated); a form
        // that is not written takes the offset of one that is (planes-only launches have no fp32 output)
        const long long o32 = out ? level_pix_off(out[0], out[l], 4, out_cs) : level_pix_off(out_hi16[0], out_hi16[l], 2, out_cs);
        const long long oh = out_hi16 ? level_pix_off(out_hi16[0], out_hi16[l], 2, out_cs) : o32;
        const long long ol = out_lo16 ? level_pix_off(out_lo16[0], out_lo16[l], 2, out_cs) : o32;
        VD3D_REQUIRE(o32 == oh && oh == ol && (out ? out[l] != nullptr : true) && o32 > (-1LL << 62),
                     "conv2d_tc16: level %d: the output forms must lie at one common pixel offset from level 0's", l);
        s.out_off[l] = o32;
        VD3D_REQUIRE((!res || res[l]) && (!res_hi16 || (res_hi16[l] && res_lo16[l])), "conv2d_tc16: level %d has no residual", l);
        if (res) {
            s.res_off[l] = level_pix_off(res[0], res[l], 4, res_cs);
            VD3D_REQUIRE(s.res_off[l] > (-1LL << 62), "conv2d_tc16: level %d: residual not at a whole-pixel offset from level 0's", l);
        }
    }
    s.w_hi = w_hi; s.w_lo = w_lo; s.out_scale = out_scale; s.bias = bias;
    s.KH = KH; s.KW = KW; s.pad = pad; s.dil = dil; s.stride = stride;
    s.res = res ? (const float*)res[0] : nullptr; s.res_cs = res_cs; s.res_co = res_co;
    s.res_h16_hi = res_hi16 ? res_hi16[0] : nullptr; s.res_h16_lo = res_lo16 ? res_lo16[0] : nullptr;
    s.out = out ? (float*)out[0] : nullptr; s.out_h16_hi = out_hi16 ? (void*)out_hi16[0] : nullptr; s.out_h16_lo = out_lo16 ? (void*)out_lo16[0] : nullptr;
    s.Cout = Cout; s.out_cs = out_cs; s.out_co = out_co; s.relu = relu; s.passes = passes; s.bn = bn;
    return conv2d_tc_launch(s, stream);
}

// The conv of vd3d_conv2d_tc16 (one tensor, stride 1) on a device list of 8 x 16 output tiles: tiles [cap] of (b, y0, x0, 0), tile_count[0] of
// them, each computed by the dense conv's K loop and epilogue (the same bits), stored only where store_map [B][Ho][Wo] is set.
extern "C" int vd3d_conv2d_tc16_tiles(const void* in_hi, const void* in_lo, int B, int H, int W, int Cin, int in_cs, int in_co,
                                      const void* w_hi, const void* w_lo, float out_scale, const float* bias, int KH, int KW, int pad, int dil,
                                      const float* res, const void* res_hi16, const void* res_lo16, int res_cs, int res_co,
                                      float* out, void* out_hi16, void* out_lo16, int Cout, int out_cs, int out_co, int relu, int bn,
                                      const int32_t* tiles, const int32_t* tile_count, const uint8_t* store_map, void* stream) {
    VD3D_REQUIRE(in_hi && in_lo && tiles && tile_count && store_map && (out || out_hi16) && (!out_hi16 == !out_lo16) && (!res_hi16 == !res_lo16) &&
                 B > 0 && H > 0 && W > 0, "conv2d_tc16_tiles: input planes, a tile list, its count, a store map and an output are required");
    VD3D_REQUIRE(((((uintptr_t)in_hi | (uintptr_t)in_lo) & 15) == 0) && ((uintptr_t)tiles & 15) == 0,
                 "conv2d_tc16_tiles: 16-byte aligned input planes and tile list are required");
    ConvSpec s;
    memset(&s, 0, sizeof(s));
    s.f16 = 1; s.L = 1; s.B = B; s.Cin = Cin; s.in_cs = in_cs; s.in_co = in_co;
    s.in[0] = in_hi; s.in_lo[0] = in_lo; s.H[0] = H; s.W[0] = W;
    s.w_hi = w_hi; s.w_lo = w_lo; s.out_scale = out_scale; s.bias = bias;
    s.KH = KH; s.KW = KW; s.pad = pad; s.dil = dil; s.stride = 1;
    s.res = res; s.res_h16_hi = res_hi16; s.res_h16_lo = res_lo16; s.res_cs = res_cs; s.res_co = res_co;
    s.out = out; s.out_h16_hi = out_hi16; s.out_h16_lo = out_lo16;
    s.Cout = Cout; s.out_cs = out_cs; s.out_co = out_co; s.relu = relu; s.passes = 3; s.bn = bn;
    s.tlist = reinterpret_cast<const int4*>(tiles); s.tcount = tile_count; s.smap = store_map;
    return conv2d_tc_launch(s, stream);
}

// ConvTranspose2d(k = 4, s = 2, p = 1) as its four sub-pixel phases, each a stride-1 2x2 conv over the H x W input, in ONE persistent launch:
//   y[b, 2m + r, 2n + s, co] = sum_{a, c in {0,1}} sum_ci x[b, m + r - 1 + a, n + s - 1 + c, ci] * Wt[ci, co, 3 - r - 2a, 3 - s - 2c]
// (rows / columns outside the input read as zero: TMA out-of-bounds fill).  Four taps of MMA work per output pixel, against 16 for a
// zero-inserted 4x4 conv.  w_hi / w_lo: [4 Cout][4 cin64] fp16, phase 2 r + s in rows (2 r + s) Cout .., k = (2 a + c) cin64 + ci
// (cin64 = Cin rounded up to 64), scaled by one power of two for all phases (out_scale undoes it).  Output [B][2H][2W][out_cs] at channel
// out_co: fp32 and / or fp16 (hi, lo) planes; epilogue bias / ReLU as vd3d_conv2d_tc16.
extern "C" int vd3d_convtranspose2d_tc16(const void* in_hi, const void* in_lo, int B, int H, int W, int Cin, int in_cs, int in_co,
                                         const void* w_hi, const void* w_lo, float out_scale, const float* bias,
                                         float* out, void* out_hi16, void* out_lo16, int Cout, int out_cs, int out_co, int relu, int bn, void* stream) {
    VD3D_REQUIRE(in_hi && in_lo && w_hi && w_lo && (out || out_hi16) && (!out_hi16 == !out_lo16) && B > 0 && H > 0 && W > 0,
                 "convtranspose2d_tc16: input planes, weights, a non-empty size and an output are required");
    VD3D_REQUIRE(Cout % 16 == 0 && Cout >= 16, "convtranspose2d_tc16: Cout must be a multiple of 16 (got %d)", Cout);
    VD3D_REQUIRE(((((uintptr_t)in_hi | (uintptr_t)in_lo) & 15) == 0), "convtranspose2d_tc16: 16-byte aligned input planes are required");
    ConvSpec s;
    memset(&s, 0, sizeof(s));
    s.f16 = 1; s.L = 4; s.convt = 1; s.B = B; s.Cin = Cin; s.in_cs = in_cs; s.in_co = in_co;
    for (int l = 0; l < 4; ++l) {
        s.in[l] = in_hi; s.in_lo[l] = in_lo; s.H[l] = H; s.W[l] = W;
        s.out_off[l] = (long long)(l >> 1) * 2 * W + (l & 1);
    }
    s.w_hi = w_hi; s.w_lo = w_lo; s.out_scale = out_scale; s.bias = bias;
    s.KH = 2; s.KW = 2; s.pad = 1; s.dil = 1; s.stride = 1;
    s.out = out; s.out_h16_hi = out_hi16; s.out_h16_lo = out_lo16;
    s.Cout = Cout; s.out_cs = out_cs; s.out_co = out_co; s.relu = relu; s.passes = 3; s.bn = bn;
    return conv2d_tc_launch(s, stream);
}

// The conv of vd3d_conv2d_tc16 (stride 1, output size = input size, fp32 output, bias, no residual / ReLU) computed only at the listed output
// pixels of each 96-column group: list [groups][B * H * W] holds counts[g] pixels b * H * W + h * W + w for group g (columns 96 g ..).
// Bit-identical to the dense conv at those pixels and columns; nothing else of `out` is written.
extern "C" int vd3d_conv2d_tc16_gather(const void* in_hi, const void* in_lo, int B, int H, int W, int Cin, int in_cs, int in_co,
                                       const void* w_hi, const void* w_lo, float out_scale, const float* bias, int KH, int KW, int pad, int dil,
                                       const int32_t* list, const int32_t* counts, int groups,
                                       float* out, int Cout, int out_cs, int out_co, void* stream) {
    VD3D_REQUIRE(in_hi && in_lo && w_hi && w_lo && list && counts && out && B > 0 && H > 0 && W > 0, "conv2d_tc16_gather: null pointer or empty input");
    VD3D_REQUIRE(KH >= 1 && KW >= 1 && dil >= 1 && 2 * pad == dil * (KH - 1) && 2 * pad == dil * (KW - 1),
                 "conv2d_tc16_gather: the output must have the input's size (2 pad = dil (K - 1), stride 1)");
    VD3D_REQUIRE(Cout % 4 == 0 && Cout >= 16 && groups == cdiv(Cout, TCG_BN) && groups <= TCG_MAX_GROUPS,
                 "conv2d_tc16_gather: Cout %d must be a multiple of 4 covered by %d groups of %d columns (<= %d groups)", Cout, groups, TCG_BN, TCG_MAX_GROUPS);
    VD3D_REQUIRE(Cin % 8 == 0 && in_cs % 8 == 0 && in_co % 8 == 0 && Cin + in_co <= in_cs && ((((uintptr_t)in_hi | (uintptr_t)in_lo) & 15) == 0),
                 "conv2d_tc16_gather: 16-byte aligned input planes with Cin, pitch and offset multiples of 8");
    VD3D_REQUIRE(out_cs % 4 == 0 && out_co % 4 == 0 && Cout + out_co <= out_cs && ((uintptr_t)out & 15) == 0 && (!bias || ((uintptr_t)bias & 7) == 0),
                 "conv2d_tc16_gather: output pitch / offset must be multiples of 4, pointers 16-byte aligned");
    VD3D_REQUIRE((long long)B * H * W < (1LL << 31), "conv2d_tc16_gather: too many pixels for the 32-bit list");
    TcParams p;
    memset(&p, 0, sizeof(p));
    p.B = B; p.H = H; p.W = W; p.Ho = H; p.Wo = W; p.Cin = Cin; p.KH = KH; p.KW = KW; p.pad = pad; p.dil = dil; p.stride = 1;
    p.Cout = Cout; p.BN = TCG_BN; p.passes = 3; p.f16 = 1; p.bk = 64; p.cin_pad = (Cin + 63) / 64 * 64; p.out_scale = out_scale;
    p.cout_pad = (Cout + 15) / 16 * 16;
    p.out_cs = out_cs; p.out_co = out_co; p.bias = bias; p.out = out;
    {
        const char* e = getenv("VD3D_TC_CHUNK");            // the dense conv's promotion chunk: the same bits
        p.chunk = e ? atoi(e) : 4;
        if (p.chunk < 1) p.chunk = 1;
    }
    TcgParams g;
    g.in_hi = (const __half*)in_hi; g.in_lo = (const __half*)in_lo; g.H = H; g.W = W; g.in_cs = in_cs; g.in_co = in_co;
    g.list = list; g.counts = counts; g.groups = groups; g.cap = B * H * W;
    g.KW = KW; g.taps = KH * KW; g.pad = pad; g.dil = dil;
    CUtensorMap mWhi, mWlo;
    int rc;
    if ((rc = make_map_wgt(&mWhi, w_hi, Cout, KH * KW * p.cin_pad, TCG_BN, 2))) return rc;
    if ((rc = make_map_wgt(&mWlo, w_lo, Cout, KH * KW * p.cin_pad, TCG_BN, 2))) return rc;
    const long long max_tiles = (long long)groups * cdiv((long long)B * H * W, 128);
    const int grid = max_tiles < kNumSMs ? (int)max_tiles : kNumSMs;
    const size_t smem = (size_t)TCG_STAGES * (2 * 128 * 128 + 2 * TCG_BN * 128) + 3 * TCG_STAGES * sizeof(uint64_t) + (TCG_MAX_GROUPS + 1) * sizeof(int) + 1024;
    const cudaError_t le = tc_launch<conv2d_tcg_kernel>(grid, TCG_THREADS, smem, stream, mWhi, mWlo, p, g);
    if (le != cudaSuccess) { set_error("conv2d_tc16_gather: launch failed: %s", cudaGetErrorString(le)); return VD3D_ECUDA; }
    VD3D_CHECK_LAUNCH("conv2d_tc16_gather");
    return VD3D_OK;
}

// ----------------------------------------------------------------------------------------------------------------
// Few-channel KHxKW convolution (the 7x7 stride-2 stem) on the tensor cores, without im2col:
// the image is kept as fp16 (hi, lo) planes [B][H][Wp][4] (<= 4 channels per pixel, `xoff` zero pixels on the left, zeros
// on the right; written by vd3d_image_to_h16_rows in row_conv.cu).  The KW*4 <= 64 values a filter row needs for output
// column wo are CONTIGUOUS in that layout, starting at pixel wo*stride (= wo*stride - pad + xoff with xoff == pad).  A tensor map with the overlapping W' stride of `stride`
// pixels therefore presents the image as a virtual NHWC tensor [B][H][Wo][64] and the conv becomes a KHx1 convolution with
// 64 "channels" (kw*4 + c; weights zero beyond KW*4) and stride (stride, 1): exactly what conv2d_tcp_kernel runs.
// ----------------------------------------------------------------------------------------------------------------
extern "C" int vd3d_stem_row_pitch(int W, int KW, int stride, int pad) {
    // pixels per padded row: left pad `pad`, the image, and enough zeros for the 16-pixel window of the last output column; even
    const int Wo = (W + 2 * pad - KW) / stride + 1;
    int need = stride * (Wo - 1) + 16;
    if (need < W + pad) need = W + pad;
    return (need + 1) / 2 * 2;
}

static int stem_launch(const void* in_hi, const void* in_lo, int B, int H, int W, int Wp, int KH, int KW, int stride, int pad, int win,
                       const void* w_hi, const void* w_lo, float out_scale, const float* bias,
                       float* out, void* out_hi16, void* out_lo16, int Cout, int out_cs, int out_co, int relu, void* stream,
                       float* pool_out, int pool_cs, int pool_co);

extern "C" int vd3d_conv2d_tc16_stem(const void* in_hi, const void* in_lo, int B, int H, int W, int Wp, int KH, int KW, int stride, int pad, int win,
                                     const void* w_hi, const void* w_lo, float out_scale, const float* bias,
                                     float* out, void* out_hi16, void* out_lo16, int Cout, int out_cs, int out_co, int relu, void* stream) {
    VD3D_REQUIRE(out, "conv2d_tc16_stem: null pointer");
    return stem_launch(in_hi, in_lo, B, H, W, Wp, KH, KW, stride, pad, win, w_hi, w_lo, out_scale, bias, out, out_hi16, out_lo16, Cout, out_cs, out_co, relu, stream,
                       nullptr, 0, 0);
}

// stem conv + BN + ReLU + MaxPool2d(3, 2, 1) in one kernel: pool_out = NHWC [B][Hp][Wp'][pool_cs], Hp = (Ho + 1) / 2, Wp' = (Wo + 1) / 2; the conv
// output itself is never written (vd3d_conv2d_tc16_stem_pool in include/vd3d_b200.h)
extern "C" int vd3d_conv2d_tc16_stem_pool(const void* in_hi, const void* in_lo, int B, int H, int W, int Wp, int KH, int KW, int stride, int pad, int win,
                                          const void* w_hi, const void* w_lo, float out_scale, const float* bias,
                                          float* pool_out, int Cout, int pool_cs, int pool_co, void* stream) {
    VD3D_REQUIRE(pool_out && Cout == 64 && pool_cs % 4 == 0 && pool_co % 4 == 0 && ((uintptr_t)pool_out & 15) == 0, "conv2d_tc16_stem_pool: 64 output channels, 16-byte aligned pooled tensor");
    return stem_launch(in_hi, in_lo, B, H, W, Wp, KH, KW, stride, pad, win, w_hi, w_lo, out_scale, bias, nullptr, nullptr, nullptr, Cout, pool_cs, pool_co, 1, stream,
                       pool_out, pool_cs, pool_co);
}

static int stem_launch(const void* in_hi, const void* in_lo, int B, int H, int W, int Wp, int KH, int KW, int stride, int pad, int win,
                       const void* w_hi, const void* w_lo, float out_scale, const float* bias,
                       float* out, void* out_hi16, void* out_lo16, int Cout, int out_cs, int out_co, int relu, void* stream,
                       float* pool_out, int pool_cs, int pool_co) {
    VD3D_REQUIRE(in_hi && in_lo && w_hi && w_lo && (out || pool_out), "conv2d_tc16_stem: null pointer");
    VD3D_REQUIRE((win == 64 || win == 32) && KW >= 1 && KW * 4 <= win && KH >= 1 && stride >= 2 && stride <= 4 && stride % 2 == 0,
                 "conv2d_tc16_stem: window of 32 or 64 elements >= 4 * KW and an even stride are required (got KW=%d win=%d stride=%d)", KW, win, stride);
    VD3D_REQUIRE(Wp == vd3d_stem_row_pitch(W, KW, stride, pad), "conv2d_tc16_stem: row pitch %d != vd3d_stem_row_pitch() = %d", Wp, vd3d_stem_row_pitch(W, KW, stride, pad));
    VD3D_REQUIRE(Cout % 16 == 0 && Cout <= 256 && out_cs % 4 == 0 && out_co % 4 == 0, "conv2d_tc16_stem: Cout must be a multiple of 16, <= 256");
    VD3D_REQUIRE(((uintptr_t)in_hi & 15) == 0 && ((uintptr_t)in_lo & 15) == 0 && ((uintptr_t)w_hi & 15) == 0 && ((uintptr_t)out & 15) == 0, "conv2d_tc16_stem: pointers must be 16-byte aligned");
    VD3D_REQUIRE(!out_hi16 || out_lo16, "conv2d_tc16_stem: fp16 output planes come in (hi, lo) pairs");
    TcParams p;
    memset(&p, 0, sizeof(p));
    p.B = B; p.H = H; p.W = W; p.Cin = win; p.KH = KH; p.KW = 1; p.pad = pad; p.dil = 1; p.stride = stride;
    p.stride_w = 1; p.pad_w = 0;
    p.Ho = (H + 2 * pad - KH) / stride + 1; p.Wo = (W + 2 * pad - KW) / stride + 1;
    VD3D_REQUIRE(p.Ho > 0 && p.Wo > 0, "conv2d_tc16_stem: empty output");
    const int BN = fit_bn(Cout);
    p.Cout = Cout; p.BN = BN; p.passes = 3; p.f16 = 1; p.bk = win; p.cin_pad = win; p.rowb = 2 * win; p.out_scale = out_scale;
    p.tiles_w = cdiv(p.Wo, TC_TW); p.tiles_h = cdiv(p.Ho, TC_TH);
    p.cout_pad = Cout;
    p.m_tiles = p.tiles_w * p.tiles_h * B; p.n_tiles = cdiv(Cout, BN);
    p.v8 = (out_cs % 8 == 0 && out_co % 8 == 0 && ((uintptr_t)out & 31) == 0 && (!bias || ((uintptr_t)bias & 31) == 0) &&
            (!out_hi16 || ((((uintptr_t)out_hi16 | (uintptr_t)out_lo16) & 15) == 0))) ? 1 : 0;
    p.out_cs = out_cs; p.out_co = out_co; p.relu = relu;
    p.bias = bias; p.out = out; p.out_h16_hi = out_hi16; p.out_h16_lo = out_lo16;
    p.range_flag = out_hi16 ? fp16_range_flag() : nullptr;
    p.chunk = 4;
    if (pool_out) {
        p.pool_out = pool_out; p.pool_cs = pool_cs; p.pool_co = pool_co;
        p.pool_H = (p.Ho + 2 - 3) / 2 + 1; p.pool_W = (p.Wo + 2 - 3) / 2 + 1;
        const long long total = (long long)B * p.pool_H * p.pool_W * (Cout / 4);
        pool_border_zero_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(pool_out, B, p.pool_H, p.pool_W, Cout / 4, pool_cs, pool_co);
        VD3D_CHECK_LAUNCH("pool_border_zero");
    }
    EncodeTiledFn enc = get_encode();
    if (!enc) { set_error("conv2d_tc16_stem: cuTensorMapEncodeTiled unavailable"); return VD3D_ECUDA; }
    CUtensorMap mA, mAlo, mWhi, mWlo;
    {
        // virtual [B][H][Wo][win] view with overlapping W' stride (stride pixels = stride * 8 bytes)
        cuuint64_t dims[4] = {(cuuint64_t)win, (cuuint64_t)p.Wo, (cuuint64_t)H, (cuuint64_t)B};
        cuuint64_t strides[3] = {(cuuint64_t)stride * 8, (cuuint64_t)Wp * 8, (cuuint64_t)H * Wp * 8};
        cuuint32_t box[4] = {(cuuint32_t)win, (cuuint32_t)TC_TW, (cuuint32_t)(TC_TH * stride), 1};
        cuuint32_t es[4] = {1, 1, (cuuint32_t)stride, 1};
        for (int i = 0; i < 2; ++i) {
            CUresult r = enc(i ? &mAlo : &mA, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, (void*)(i ? in_lo : in_hi), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                             win == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) { set_error("conv2d_tc16_stem: cuTensorMapEncodeTiled(image) failed: %d", (int)r); return VD3D_ECUDA; }
        }
    }
    int rc;
    if ((rc = make_map_wgt(&mWhi, w_hi, Cout, KH * win, BN, 2, 2 * win))) return rc;
    if ((rc = make_map_wgt(&mWlo, w_lo, Cout, KH * win, BN, 2, 2 * win))) return rc;
    return tcp_launch(p, mA, mAlo, mWhi, mWlo, stream);
}

extern "C" int vd3d_split_lo_nhwc(const float* in, float* lo, long long npix, int C, int cs, int co, void* stream) {
    VD3D_REQUIRE(in && lo && C % 4 == 0 && cs % 4 == 0 && co % 4 == 0, "split_lo: bad args");
    long long total = npix * (C / 4);
    split_lo_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(in, lo, npix, C / 4, cs, co);
    VD3D_CHECK_LAUNCH("split_lo");
    return VD3D_OK;
}

extern "C" int vd3d_split_h16_nhwc(const float* in, void* hi16, void* lo16, long long npix, int C, int cs, int co, void* stream) {
    VD3D_REQUIRE(in && hi16 && lo16 && C % 4 == 0 && cs % 4 == 0 && co % 4 == 0, "split_h16: bad args");
    long long total = npix * (C / 4);
    split_h16_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(in, (__half*)hi16, (__half*)lo16, npix, C / 4, cs, co, fp16_range_flag());
    VD3D_CHECK_LAUNCH("split_h16");
    return VD3D_OK;
}
