// PSMCosine cost volume (R/lib/PSM_cost_volume.py:76-91) on the Hopper tensor cores (wgmma).
//
//   cost[q, d] = (x(q) >= d) ? 1/C * sum_c L[q, c] * R[q - d, c] : 0        q = flat pixel index (b, y, x), x(q) = q mod W
//
// The SIMT kernels of cost_volume.cu are bound by shared-memory reads and instruction issue; the correlation is a banded matrix product,
// so here it is computed as the FULL product of a 128-pixel L tile with the 160-pixel R window [q0 - 32, q0 + 128) on the tensor core and
// only the band is kept:
//
//   * pixels are addressed flat across rows and images: R[q - d] leaves the row exactly when x(q) < d, where the reference
//     writes 0, so the tile grid needs no row alignment (B*H*W / 128 tiles, no ragged tiles at W = 320).
//   * operands are the fp16 (hi, lo) planes the tensor-core convs already produce for the features; three kind::f16 MMAs per
//     k-step (Llo*Rhi + Lhi*Rlo + Lhi*Rhi) into one fp32 accumulator [128 x 160]: 22 significant operand bits, and only
//     4 * C/64 * 3 accumulations, so no promotion is needed (error ~1e-6 of the 1e-3 parity budget).
//   * warp 8 = TMA producer (4 boxes per 64-channel k-block: Lhi, Llo [128 x 64], Rhi, Rlo [160 x 64], 128-byte swizzle),
//     warps 0..7 = two consumer warpgroups (64 L pixels x 160 window pixels each): after the last k-block every thread parks the
//     accumulator entries of the band (window pixel - L pixel in [0, 32]) in a [128][36] shared-memory tile, then thread t writes the
//     disparities d = 4 (t / 128) + 8 i of pixel t % 128: scale, mask, 16-byte stores.
//   * persistent: one CTA per SM strides over the tiles; HBM traffic = the algorithmic bytes (each L / R element once from
//     DRAM, the 32-pixel window overlap comes from L2).
#include "tc_common.cuh"
#include <cstring>

namespace vd3d {

constexpr int PT_M = 128;                 // L pixels per tile
constexpr int PT_PAD = 32;                // R window starts PT_PAD pixels before the tile: disparities < 32
constexpr int PT_N = PT_M + PT_PAD;       // 160 R pixels (wgmma N)
constexpr int PT_THREADS = 256 + 32;      // warps 0..7 = consumers, warp 8 = TMA producer
constexpr int PT_STAGES = 2;
constexpr int PT_L_BYTES = PT_M * 128, PT_R_BYTES = PT_N * 128;
constexpr int PT_STAGE_BYTES = 2 * PT_L_BYTES + 2 * PT_R_BYTES;       // 73728
constexpr int PT_BAND_LD = 36;                                          // band tile row: entries 0..32 used

struct PsmTcParams {
    long long npix;
    int W, D, kblocks, ntiles;
    int out_cs, out_co;
    float inv_c;
    float* out;
};

__global__ void __launch_bounds__(PT_THREADS, 1)
psm_cosine_tc_kernel(const __grid_constant__ CUtensorMap mapLhi, const __grid_constant__ CUtensorMap mapLlo,
                     const __grid_constant__ CUtensorMap mapRhi, const __grid_constant__ CUtensorMap mapRlo, const PsmTcParams p) {
    extern __shared__ __align__(1024) uint8_t psm_tc_smem[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(psm_tc_smem) + 1023) & ~(uintptr_t)1023);
    float* band = reinterpret_cast<float*>(smem + (size_t)PT_STAGES * PT_STAGE_BYTES);
    uint64_t* full = reinterpret_cast<uint64_t*>(band + PT_M * PT_BAND_LD);     // [stages]  TMA -> consumers
    uint64_t* empty = full + PT_STAGES;                                          // [stages]  consumers (8 warps) -> TMA

    const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < PT_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            // ================= TMA producer =================
            int it = 0;
            for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
                const int q0 = tile * PT_M;                     // npix < 2^31 (checked on the host)
                for (int kb = 0; kb < p.kblocks; ++kb, ++it) {
                    const int s = it % PT_STAGES, ph = (it / PT_STAGES) & 1;
                    mbar_wait(&empty[s], ph ^ 1);
                    uint8_t* st = smem + (size_t)s * PT_STAGE_BYTES;
                    mbar_expect_tx(&full[s], PT_STAGE_BYTES);
                    tma_load_2d(st, &mapLhi, &full[s], kb * 64, q0);
                    tma_load_2d(st + PT_L_BYTES, &mapLlo, &full[s], kb * 64, q0);
                    tma_load_2d(st + 2 * PT_L_BYTES, &mapRhi, &full[s], kb * 64, q0 - PT_PAD);         // rows < 0: zero fill (masked anyway)
                    tma_load_2d(st + 2 * PT_L_BYTES + PT_R_BYTES, &mapRlo, &full[s], kb * 64, q0 - PT_PAD);
                }
            }
        }
    } else {
        // ================= consumer warpgroups =================
        const int wg = warp >> 2;
        auto release = [&](int st) {
            __syncwarp();
            if (st >= 0 && lane == 0) mbar_arrive(&empty[st]);
        };
        float acc[PT_N / 2];
        int it = 0;
        const int t = warp * 32 + lane, row = t & (PT_M - 1), dh = t >> 7;
        for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
            int pend = -1;
            for (int kb = 0; kb < p.kblocks; ++kb, ++it) {
                const int s = it % PT_STAGES, ph = (it / PT_STAGES) & 1;
                mbar_wait(&full[s], ph);
                const uint32_t sa = smem_u32(smem + (size_t)s * PT_STAGE_BYTES);
                const uint32_t la = sa + (uint32_t)wg * 64u * 128u;
                const uint64_t dLh = make_sdesc(la), dLl = make_sdesc(la + PT_L_BYTES);
                const uint64_t dRh = make_sdesc(sa + 2 * PT_L_BYTES), dRl = make_sdesc(sa + 2 * PT_L_BYTES + PT_R_BYTES);
                wg_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const uint64_t off = (uint64_t)((k * 32) >> 4);
                    wgmma_f16<PT_N>(acc, dLl + off, dRh + off, (kb == 0 && k == 0) ? 0u : 1u);
                    wgmma_f16<PT_N>(acc, dLh + off, dRl + off, 1u);
                    wgmma_f16<PT_N>(acc, dLh + off, dRh + off, 1u);
                }
                wg_commit();
                wg_wait<1>();                                  // the previous k-block's MMAs are done
                release(pend); pend = s;
            }
            wg_wait<0>();                                      // (outside the loop: a drain under a branch in it would make ptxas drain every k-block)
            release(pend);
            wg_fence_regs(acc);
            consumers_sync();                                  // the previous tile's band has been read
            {
                const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
                for (int j = 0; j < PT_N / 8; ++j)
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const int r = r0 + 8 * (e >> 1), k = 8 * j + c0 + (e & 1) - r;      // window pixel - L pixel
                        if (k >= 0 && k <= PT_PAD) band[r * PT_BAND_LD + k] = acc[4 * j + e];
                    }
            }
            consumers_sync();
            const long long pix = (long long)tile * PT_M + row;
            if (pix < p.npix) {
                const int x = (int)(pix % p.W);
                float* op = p.out + pix * p.out_cs + p.out_co;
                const float* bp = band + row * PT_BAND_LD;
                // disparity d <-> window pixel row - d + 32 <-> band entry 32 - d
                for (int d = 4 * dh; d < p.D; d += 8) {
                    float4 o;
                    o.x = (x >= d + 0) ? bp[32 - d] * p.inv_c : 0.f;
                    o.y = (x >= d + 1) ? bp[31 - d] * p.inv_c : 0.f;
                    o.z = (x >= d + 2) ? bp[30 - d] * p.inv_c : 0.f;
                    o.w = (x >= d + 3) ? bp[29 - d] * p.inv_c : 0.f;
                    *reinterpret_cast<float4*>(op + d) = o;
                }
            }
        }
    }
}

}  // namespace vd3d

using namespace vd3d;

extern "C" int vd3d_psm_cosine_h16(const void* l_hi, const void* l_lo, const void* r_hi, const void* r_lo, long long npix, int W, int C,
                                   int cs, int co, int D, float* out, int out_cs, int out_co, void* stream) {
    VD3D_REQUIRE(l_hi && l_lo && r_hi && r_lo && out, "psm_cosine_h16: null pointer");
    VD3D_REQUIRE(npix > 0 && npix < (1ll << 31) - 256 && W > 0, "psm_cosine_h16: bad sizes");
    VD3D_REQUIRE(C % 64 == 0 && C > 0, "psm_cosine_h16: C must be a multiple of 64 (got %d)", C);
    VD3D_REQUIRE(D > 0 && D <= PT_PAD && D % 4 == 0, "psm_cosine_h16: D must be a multiple of 4 in [4, 32] (got %d)", D);
    VD3D_REQUIRE(cs % 8 == 0 && co % 8 == 0 && cs >= co + C, "psm_cosine_h16: feature pitch/offset must be multiples of 8");
    VD3D_REQUIRE(out_cs % 4 == 0 && out_co % 4 == 0 && out_cs >= out_co + D, "psm_cosine_h16: output pitch/offset must be multiples of 4");
    VD3D_REQUIRE((((uintptr_t)l_hi | (uintptr_t)l_lo | (uintptr_t)r_hi | (uintptr_t)r_lo | (uintptr_t)out) & 15) == 0, "psm_cosine_h16: pointers must be 16-byte aligned");
    PsmTcParams p;
    memset(&p, 0, sizeof(p));
    p.npix = npix; p.W = W; p.D = D; p.kblocks = C / 64; p.ntiles = (int)((npix + PT_M - 1) / PT_M);
    p.out_cs = out_cs; p.out_co = out_co; p.inv_c = 1.0f / (float)C; p.out = out;
    CUtensorMap mLh, mLl, mRh, mRl;
    int rc;
    const __half* lh = (const __half*)l_hi + co; const __half* ll = (const __half*)l_lo + co;
    const __half* rh = (const __half*)r_hi + co; const __half* rl = (const __half*)r_lo + co;
    if ((rc = make_map_2d_h16(&mLh, lh, npix, C, cs, PT_M, "psm_cosine_h16"))) return rc;
    if ((rc = make_map_2d_h16(&mLl, ll, npix, C, cs, PT_M, "psm_cosine_h16"))) return rc;
    if ((rc = make_map_2d_h16(&mRh, rh, npix, C, cs, PT_N, "psm_cosine_h16"))) return rc;
    if ((rc = make_map_2d_h16(&mRl, rl, npix, C, cs, PT_N, "psm_cosine_h16"))) return rc;
    const size_t smem = (size_t)PT_STAGES * PT_STAGE_BYTES + PT_M * PT_BAND_LD * sizeof(float) + 2 * PT_STAGES * sizeof(uint64_t) + 1024;
    static bool attr_set = false;
    if (!attr_set) {
        VD3D_CUDA(cudaFuncSetAttribute(psm_cosine_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        attr_set = true;
    }
    const int grid = p.ntiles < kNumSMs ? p.ntiles : kNumSMs;
    psm_cosine_tc_kernel<<<grid, PT_THREADS, smem, (cudaStream_t)stream>>>(mLh, mLl, mRh, mRl, p);
    VD3D_CHECK_LAUNCH("psm_cosine_h16");
    return VD3D_OK;
}
