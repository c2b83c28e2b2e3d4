// 64 -> 64-channel 3x3 / stride-1 / pad-1 convolutions (ResNet layer1, DLA-34's level-2 blocks) of the fp16-split engine as a ROW-STRIP kernel:
// bit-identical to conv2d_tcp_kernel (conv2d_tc.cu), with every input row staged once and the epilogue overlapped on seven warps.
//
// * Tile = two output rows x 64 columns.  Warpgroup w issues the m64 MMAs of output row 2t + w, so its 64 A rows are 64 consecutive pixels.
//   A CTA walks down a 64-column strip of one image: the (image, strip, row pair) tiles are numbered strip-major and every CTA takes one
//   contiguous run of them (at most one more tile than any other CTA), so it restarts the row stream at most once per strip it enters.
// * Input rows, staged once: output rows 2t, 2t + 1 read input rows 2t - 1 .. 2t + 2, two of which the next tile reads again, so the producer
//   streams two new rows per tile into a ring of R64_RING rows.  A staged row is 66 pixels (one halo column on each side) x 64 channels, hi and
//   lo, in no-swizzle core-matrix order: 8-channel group j of pixel x at byte j * R64_PLANE + 16 x (a 5-D TMA box {8 ch, 66 px, 8 groups, 1, 1};
//   the conv's zero padding, the halo columns beyond the image and channels >= Cin are TMA out-of-bounds fill).  A K-major no-swizzle wgmma
//   operand is 8-row x 16-byte core matrices, so the descriptor (leading byte offset R64_PLANE between the two 8-channel groups of a K step,
//   stride byte offset 128 between 8-pixel groups) reads operand row m of tap (ky, kx) at staged pixel m + kx of row 2t + w + ky: the window
//   shift is 16 kx bytes and nothing is re-read or re-laid-out.
// * Weights: one [BN][64] hi | lo k-block (SWIZZLE_128B, as conv2d_tcp_kernel) per tap, streamed through a ring in the same tap order every
//   tile (L2-resident).
// * MMAs: exactly conv2d_tcp_kernel's sequence: K order tap 0..8 (one 64-channel chunk), promotion chunks of p.chunk k-blocks, the three
//   products of wg_kblock in the same order (wg_tile_kloop), so every output element sees the same wgmma chain and gets the same bits.
// * Epilogue: the consumers stage each tile's accumulator ([128][BN + 4] fp32, outside the rings) and hand it to the seven epilogue warps
//   through acc_full / acc_empty, then go on with the next tile's MMAs.  Per element the arithmetic is tcp_epi_res / tcp_epi_out.
//
// Warps 0..7 = two consumer warpgroups, warp 8 = TMA producer, warps 9..15 = epilogue.  512 threads: the 128-register budget per thread is
// enough for the 64-column consumers (no setmaxnreg).
//
// Shared memory (BN = 64): weight ring 5 x 16 KB + row ring 6 x 16.5 KB + staged tile 34 KB + barriers = 214 KB of the 227 KB.
#include "tc_conv.cuh"
#include <cstring>

namespace vd3d {

constexpr int R64_PX = 64;                            // output columns per strip
constexpr int R64_ROWPX = R64_PX + 2;                 // staged pixels per input row
constexpr uint32_t R64_PLANE = R64_ROWPX * 16;        // bytes of one 8-channel group of a staged row (core-matrix rows 16 bytes apart)
constexpr uint32_t R64_ROWB = 8 * R64_PLANE;          // bytes of a staged row per fp16 plane (8448; a multiple of 128 as TMA needs)
constexpr uint32_t R64_SLOT = 2 * R64_ROWB;           // [hi | lo]
constexpr int R64_RING = 6;                           // the 4 rows of the current tile and the next tile's 2
constexpr int R64_EPI = 224;                          // epilogue threads (7 warps)
constexpr int R64_THREADS = TC_CONSUMERS + 32 + R64_EPI;
constexpr int R64_MAX_WST = 8;

struct R64Geo {
    int nstrips, rpairs;                              // strips per image row, output row pairs per image
    long long ntiles;                                 // B * nstrips * rpairs
    int wstages;                                      // weight ring stages
};

__device__ __forceinline__ void tma_load_5d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3, int c4) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(smem_u32(dst)),
        "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
        : "memory");
}

// Run of tiles [t0, t1) of one strip: image b, strip s, first output row pair rp0 (tiles are numbered (b, s, row pair), row pair fastest)
struct R64Run { int b, s, rp0, T; };
__device__ __forceinline__ R64Run r64_run(const R64Geo& q, long long t0, long long t1) {
    R64Run r;
    const long long bs = t0 / q.rpairs;
    r.rp0 = (int)(t0 - bs * q.rpairs);
    r.s = (int)(bs % q.nstrips); r.b = (int)(bs / q.nstrips);
    r.T = (int)min((long long)(q.rpairs - r.rp0), t1 - t0);
    return r;
}

__device__ __forceinline__ void r64_epilogue_sync() { asm volatile("bar.sync 3, %0;" ::"n"(R64_EPI) : "memory"); }

template <int BN>
__global__ void __launch_bounds__(R64_THREADS, 1)
conv2d_row64_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapAlo,
                    const __grid_constant__ CUtensorMap mapWhi, const __grid_constant__ CUtensorMap mapWlo, const TcParams p, const R64Geo q) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    constexpr int LD = BN + 4;
    constexpr uint32_t WB = (uint32_t)BN * 128u;                      // one weight plane of a tap
    constexpr uint32_t WSTAGE = 2u * WB;                              // [W hi | W lo]
    uint8_t* const wring = smem;                                      // [wstages] (1024-aligned: SWIZZLE_128B)
    uint8_t* const rring = wring + (size_t)q.wstages * WSTAGE;        // [R64_RING]
    float* const tile = reinterpret_cast<float*>(rring + (size_t)R64_RING * R64_SLOT);
    uint64_t* const rfull = reinterpret_cast<uint64_t*>(tile + 128 * LD);   // [R64_RING]  TMA -> consumers
    uint64_t* const rempty = rfull + R64_RING;                        // [R64_RING]  consumers (8 warps) -> producer
    uint64_t* const wfull = rempty + R64_RING;                        // [wstages]
    uint64_t* const wempty = wfull + R64_MAX_WST;                     // [wstages]
    uint64_t* const acc_full = wempty + R64_MAX_WST;                  // consumers (256 threads) -> epilogue: a tile is staged
    uint64_t* const acc_empty = acc_full + 1;                         // epilogue -> consumers: the staged tile has been read

    const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
    const long long t_lo = (long long)blockIdx.x * q.ntiles / gridDim.x, t_hi = (long long)(blockIdx.x + 1) * q.ntiles / gridDim.x;

    if (threadIdx.x == 0) {
        for (int s = 0; s < R64_RING; ++s) { mbar_init(&rfull[s], 1); mbar_init(&rempty[s], TC_CONSUMERS / 32); }
        for (int s = 0; s < q.wstages; ++s) { mbar_init(&wfull[s], 1); mbar_init(&wempty[s], TC_CONSUMERS / 32); }
        mbar_init(acc_full, TC_CONSUMERS);
        mbar_init(acc_empty, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    pdl_launch_dependents();
    pdl_wait();

    if (warp > TC_CONSUMERS / 32) {
        // ================= epilogue warps: tile i of this CTA is handed over through acc_full / acc_empty phase i =================
        constexpr int CG = BN / 8;                                    // 8-channel groups per pixel
        constexpr int ITEMS = 128 * CG;
        constexpr int U = (ITEMS + R64_EPI - 1) / R64_EPI;            // items per thread: all residual loads in flight before the first output
        const int et = (int)threadIdx.x - (TC_CONSUMERS + 32);
        float amax = 0.f;
        int i = 0;
        for (long long t0 = t_lo; t0 < t_hi;) {
            const R64Run run = r64_run(q, t0, t_hi);
            t0 += run.T;
            for (int t = 0; t < run.T; ++t, ++i) {
                mbar_wait(acc_full, i & 1);
                if (!(p.dbg & 16)) {
                    const int ho0 = 2 * (run.rp0 + t), wo0 = run.s * R64_PX;
                    // item = r * CG + g (pixel row r of the staged tile, channel group g): consecutive lanes on consecutive groups of one pixel
                    float rr[U][8];
                    long long pix[U];
                    int it[U];
#pragma unroll
                    for (int k = 0; k < U; ++k) {
                        const int idx = et + k * R64_EPI;
                        const int r = idx / CG, g = idx - r * CG;
                        const int ho = ho0 + (r >> 6), wo = wo0 + (r & 63);
                        it[k] = (idx < ITEMS && ho < p.Ho && wo < p.Wo && 8 * g + 4 <= p.Cout) ? idx : -1;
                        pix[k] = ((long long)run.b * p.Ho + ho) * p.Wo + wo;
                        if (it[k] >= 0) tcp_epi_res(p, pix[k], 8 * g, rr[k]);
                    }
#pragma unroll
                    for (int k = 0; k < U; ++k) {
                        if (it[k] < 0) continue;
                        const int r = it[k] / CG, g = it[k] - r * CG;
                        const float* acc = tile + r * LD + 8 * g;
                        const float4 a0 = *reinterpret_cast<const float4*>(acc), a1 = *reinterpret_cast<const float4*>(acc + 4);
                        amax = fmaxf(amax, tcp_epi_out(p, pix[k], 8 * g, a0, a1, rr[k]));
                    }
                }
                r64_epilogue_sync();                                  // every epilogue thread is done reading the staged tile
                if (et == 0) mbar_arrive(acc_empty);
            }
        }
        note_fp16_range(amax, p.range_flag);
    } else if (warp == TC_CONSUMERS / 32) {
        // ================= TMA producer: per tile the rows not yet staged, then the 9 weight k-blocks =================
        if (lane == 0) {
            int gl = 0;                                               // ring index of the current run's first row
            int ws = 0, wph = 0;                                      // weight slot and its fill parity
            for (long long t0 = t_lo; t0 < t_hi;) {
                const R64Run run = r64_run(q, t0, t_hi);
                t0 += run.T;
                const int yi0 = 2 * run.rp0 - 1, xi0 = run.s * R64_PX - 1;      // input row / column of the run's staged row 0, pixel 0
                for (int t = 0; t < run.T; ++t) {
                    for (int l = (t == 0 ? 0 : 2 * t + 2); l < 2 * t + 4; ++l) {
                        const int g = gl + l, slot = g % R64_RING;
                        mbar_wait(&rempty[slot], ((g / R64_RING) & 1) ^ 1);
                        uint8_t* dst = rring + (size_t)slot * R64_SLOT;
                        mbar_expect_tx(&rfull[slot], R64_SLOT);
                        tma_load_5d(dst, &mapA, &rfull[slot], 0, xi0, 0, yi0 + l, run.b);
                        tma_load_5d(dst + R64_ROWB, &mapAlo, &rfull[slot], 0, xi0, 0, yi0 + l, run.b);
                    }
                    for (int tap = 0; tap < 9; ++tap) {
                        mbar_wait(&wempty[ws], wph ^ 1);
                        uint8_t* dst = wring + (size_t)ws * WSTAGE;
                        mbar_expect_tx(&wfull[ws], WSTAGE);
                        tma_load_2d(dst, &mapWhi, &wfull[ws], tap * 64, 0);
                        tma_load_2d(dst + WB, &mapWlo, &wfull[ws], tap * 64, 0);
                        if (++ws == q.wstages) { ws = 0; wph ^= 1; }
                    }
                }
                gl += 2 * run.T + 2;
            }
        }
    } else {
        // ================= consumer warpgroups: MMAs of output row 2t + wg, chunk promotion, hand-off to the epilogue =================
        const int wg = warp >> 2;
        const uint32_t rbase = smem_u32(rring), wbase = smem_u32(wring);
        int ws = 0, wph = 0;
        int row0 = 0, tap = 0;                                        // ring index of the tile's first staged row; next k-block's tap
        auto acquire = [&]() {
            mbar_wait(&wfull[ws], wph);
            const int ky = tap / 3, kx = tap - 3 * ky;
            ++tap;
            const uint32_t ra = rbase + (uint32_t)((row0 + wg + ky) % R64_RING) * R64_SLOT + 16u * (uint32_t)kx;
            const uint32_t wa = wbase + (uint32_t)ws * WSTAGE;
            const KbOperands o{make_sdesc_ns(ra, R64_PLANE, 128u), make_sdesc_ns(ra + R64_ROWB, R64_PLANE, 128u), make_sdesc(wa), make_sdesc(wa + WB), ws};
            if (++ws == q.wstages) { ws = 0; wph ^= 1; }
            return o;
        };
        auto release = [&](int slot) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&wempty[slot]);
        };
        auto release_row = [&](int g) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&rempty[g % R64_RING]);
        };
        auto issued = [&]() {};
        float tot[BN / 2], c[BN / 2];
        int gl = 0, i = 0;
        for (long long t0 = t_lo; t0 < t_hi;) {
            const R64Run run = r64_run(q, t0, t_hi);
            t0 += run.T;
            for (int t = 0; t < run.T; ++t, ++i) {
                row0 = gl + 2 * t;
                for (int l = (t == 0 ? 0 : 2 * t + 2); l < 2 * t + 4; ++l) mbar_wait(&rfull[(gl + l) % R64_RING], ((gl + l) / R64_RING) & 1);
#pragma unroll
                for (int k = 0; k < BN / 2; ++k) tot[k] = 0.f;
                tap = 0;
                // 2 * R64_PLANE / 16: a K step (16 channels) moves two 8-channel groups
                wg_tile_kloop<BN, true, 0, 4, 2 * (int)R64_PLANE / 16>(tot, c, 9, p.chunk, acquire, release, issued);
                release_row(row0); release_row(row0 + 1);            // the next tile reads rows 2t + 2 .. 2t + 5
                // the epilogue is done with the previous staged tile (phase i - 1 of acc_empty; a fresh barrier passes parity 1)
                mbar_wait(acc_empty, (i & 1) ^ 1);
                wg_stage<BN>(tot, tile, LD, wg, warp, lane);
                mbar_arrive(acc_full);
            }
            release_row(gl + 2 * run.T); release_row(gl + 2 * run.T + 1);
            gl += 2 * run.T + 2;
        }
    }
}

// The conv of `p` (set up by conv2d_tc_launch, eligible per conv2d_row64_eligible) on the row-strip kernel.  Input planes: NHWC fp16 with
// pixel pitch in_cs, channel offset in_co.
int conv2d_row64_launch(TcParams& p, const void* in_hi, const void* in_lo, int in_cs, int in_co, const void* w_hi, const void* w_lo, void* stream) {
    const int BN = p.BN;
    VD3D_REQUIRE(conv2d_row64_eligible(p), "conv2d_row64: not a 64-channel 3x3 / stride-1 / pad-1 fp16-split conv with one output tile");
    { const char* e = getenv("VD3D_TC_DEBUG"); p.dbg = e ? atoi(e) : 0; }
    p.trace = nullptr; p.trace_n = 0;
    EncodeTiledFn enc = get_encode();
    if (!enc) { set_error("conv2d_row64: cuTensorMapEncodeTiled unavailable"); return VD3D_ECUDA; }
    CUtensorMap mA, mAlo, mWhi, mWlo;
    {
        // [B][H][8-channel group][W][8]: the box {8, 66, 8, 1, 1} lands as 8 planes of 66 pixels x 16 bytes
        cuuint64_t dims[5] = {8, (cuuint64_t)p.W, (cuuint64_t)(p.Cin / 8), (cuuint64_t)p.H, (cuuint64_t)p.B};
        cuuint64_t strides[4] = {(cuuint64_t)in_cs * 2, 16, (cuuint64_t)p.W * in_cs * 2, (cuuint64_t)p.H * p.W * in_cs * 2};
        cuuint32_t box[5] = {8, (cuuint32_t)R64_ROWPX, 8, 1, 1};
        cuuint32_t es[5] = {1, 1, 1, 1, 1};
        for (int i = 0; i < 2; ++i) {
            const char* base = (const char*)(i ? in_lo : in_hi) + (size_t)in_co * 2;
            const CUresult r = enc(i ? &mAlo : &mA, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, (void*)base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                   CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) { set_error("conv2d_row64: cuTensorMapEncodeTiled(activation) failed: %d", (int)r); return VD3D_ECUDA; }
        }
    }
    int rc;
    if ((rc = make_map_wgt(&mWhi, w_hi, p.Cout, 9 * 64, BN, 2))) return rc;
    if ((rc = make_map_wgt(&mWlo, w_lo, p.Cout, 9 * 64, BN, 2))) return rc;
    R64Geo q;
    q.nstrips = cdiv(p.Wo, R64_PX); q.rpairs = cdiv(p.Ho, 2);
    q.ntiles = (long long)p.B * q.nstrips * q.rpairs;
    const size_t wstage = (size_t)2 * BN * 128;
    const size_t fixed = (size_t)R64_RING * R64_SLOT + (size_t)128 * (BN + 4) * sizeof(float) + (2 * R64_RING + 2 * R64_MAX_WST + 2) * sizeof(uint64_t) + 1024;
    const size_t avail = 227 * 1024;
    q.wstages = (int)((avail - fixed) / wstage);
    if (q.wstages > R64_MAX_WST) q.wstages = R64_MAX_WST;
    VD3D_REQUIRE(q.wstages >= 3, "conv2d_row64: shared-memory budget exceeded");
    const size_t smem = fixed + q.wstages * wstage;
    int grid = q.ntiles < kNumSMs ? (int)q.ntiles : kNumSMs;
    { const char* e = getenv("VD3D_TC_GRID"); const int cap = e ? atoi(e) : 0; if (cap > 0 && cap < grid) grid = cap; }     // diagnostics
    cudaError_t le = cudaErrorInvalidValue;
    switch (BN) {
        case 16: le = tc_launch<conv2d_row64_kernel<16>>(grid, R64_THREADS, smem, stream, mA, mAlo, mWhi, mWlo, p, q); break;
        case 32: le = tc_launch<conv2d_row64_kernel<32>>(grid, R64_THREADS, smem, stream, mA, mAlo, mWhi, mWlo, p, q); break;
        case 48: le = tc_launch<conv2d_row64_kernel<48>>(grid, R64_THREADS, smem, stream, mA, mAlo, mWhi, mWlo, p, q); break;
        case 64: le = tc_launch<conv2d_row64_kernel<64>>(grid, R64_THREADS, smem, stream, mA, mAlo, mWhi, mWlo, p, q); break;
    }
    if (le != cudaSuccess) { set_error("conv2d_row64: launch failed: %s", cudaGetErrorString(le)); return VD3D_ECUDA; }
    VD3D_CHECK_LAUNCH("conv2d_row64");
    return VD3D_OK;
}

}  // namespace vd3d
