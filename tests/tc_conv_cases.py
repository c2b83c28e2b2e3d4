"""Constructed cases for the fp16-split tensor-core conv engine (csrc/conv2d_tc.cu, csrc/tc_conv.cuh, csrc/conv2d_row64.cu), its float64
references, and host restatements of the launch choices conv2d_tc_launch / tcp_launch make.

Entries under test: vd3d_conv2d_tc16 (one level and multi-level launches; 64-channel 3x3 convs go to the row-strip kernel),
vd3d_convtranspose2d_tc16 (the four sub-pixel phases as four levels of one launch) and the 3xTF32 vd3d_conv2d_tc.

Every case row names the path it reaches as a string: "BN=<tile width> <staging> v8=<0|1>" for conv2d_tcp_kernel, where staging is "sep"
(a separate staging tile after the operand ring), "ring" (the accumulator staged in the stage of the tile's last k-block) or "split" (ring,
rows 64..127 in a half tile); "BN=<w> v8=<0|1> row64" for the row-strip kernel; plus " mblock=<n>" for an L2-blocked tile order and
" L=<levels>" for multi-level launches.  `reach` restates the host code, so a row edited off its path fails the CPU test.

Operands come in two kinds:
  * exact: integer activations in [-4, 4], weights m / 8 with |m| <= 8 (max |w| = 1, so fp16_split_scaled scales by 2^14 and every scaled
    weight is a whole fp16 with lo = 0), bias m / 8 in [-2, 2], residual integers in [-8, 8].  Every product and partial sum lies on the
    grid 1/8 (2^11 after the weight scale) far below 2^20 grid units, so the truncating tensor-core accumulator adds them exactly: the result
    does not depend on tile order, chunking or the accumulation model and must equal float64 bit for bit.  The planes are built directly,
    one family per plane product: (a) x_hi, w_hi; (b) x_lo with x_hi = 0; (c) w_lo with w_hi = 0; (d) x_lo and w_lo only, the product
    the engine drops by design (the output is then exactly bias + residual);
  * normal: random normals, compared with the per-element bound `tc16_bound` / `tf32_bound` (below).
"""
import math
from collections import namedtuple

import torch
import torch.nn.functional as F

# ---------------------------------------------------------------------------------------------------------------------------------------
# host restatement of the launch choices (csrc/conv2d_tc.cu: conv2d_tc_launch, tcp_launch; csrc/tc_conv.cuh: conv2d_row64_eligible)
# ---------------------------------------------------------------------------------------------------------------------------------------
TC_TW, TC_TH = 16, 8
TC_MAX_BN = 128
TC_MAX_LEVELS = 5
NUM_SMS = 132
SMEM_AVAIL = 227 * 1024 - 1024 - 256


def cdiv(a, b):
    return (a + b - 1) // b


def pick_bn_persistent(Cout):
    """vd3d_tc_pick_bn_persistent: the widest tile <= 128 that splits Cout evenly into 16-column granules"""
    cp = cdiv(Cout, 16) * 16
    nt = cdiv(cp, TC_MAX_BN)
    return cdiv(cdiv(cp, nt), 16) * 16


def pick_bn_cost(Cout, m_tiles):
    """the fp16-split engine's default tile width: minimise rounds x (BN + 64) over 16-column granules, ties to the wider tile"""
    cp = cdiv(Cout, 16) * 16
    if cp <= TC_MAX_BN:
        return cp
    best, best_cost = pick_bn_persistent(Cout), -1
    for bn in range(64, TC_MAX_BN + 1, 16):
        cost = cdiv(m_tiles * cdiv(cp, bn), NUM_SMS) * (bn + 64)
        if best_cost < 0 or cost < best_cost or (cost == best_cost and bn > best):
            best, best_cost = bn, cost
    return best


def pick_bn_tf32(Cout):
    """vd3d_tc_pick_bn: the 3xTF32 engine's default tile width"""
    if Cout % 128 == 0:
        return 128
    if Cout < 128 and Cout % 16:
        return cdiv(Cout, 16) * 16
    for bn in (96, 64, 48, 32):
        if Cout % bn == 0:
            return bn
    return cdiv(Cout, 16) * 16 if Cout <= 128 else 128


def fit_bn(bn):
    """a requested tile wider than 128 runs as equal halves of 16-column granules"""
    while bn > TC_MAX_BN:
        bn = cdiv(bn // 2, 16) * 16
    return bn


def tcp_epi_warps(BN):
    return BN > 64


def tile_ld(BN):
    return BN if BN == TC_MAX_BN else BN + 4


def ring_layout(BN, tile_in_ring_env=None, rowb=128):
    """(stages, tile_in_ring, split_stage) of tcp_launch"""
    stage = 2 * 128 * rowb + 2 * BN * rowb
    tile = 128 * tile_ld(BN) * 4
    stages = (SMEM_AVAIL - tile) // stage
    stages_in = SMEM_AVAIL // stage
    in_ring = not (tile_in_ring_env is not None and int(tile_in_ring_env) == 0) and tile <= stage and stages < 8 and stages_in > stages
    if in_ring:
        stages = stages_in
    stages = min(stages, 8)
    split = in_ring and tcp_epi_warps(BN) and stages * stage + tile // 2 <= SMEM_AVAIL
    return stages, in_ring, split


def mblock(m_tiles, n_tiles, stride, cin_pad, f16, l2mb=20.0):
    """scheduling units per M block of the L2-aware tile order (0: one block)"""
    if n_tiles <= 1 or l2mb <= 0:
        return 0
    mb = max(8, int(l2mb * 1048576.0 / (128.0 * stride * stride * cin_pad * (4.0 if f16 else 8.0))))
    if mb >= m_tiles:
        return 0
    return cdiv(m_tiles, cdiv(m_tiles, mb))


def v8_ok(out_cs, out_co, bias_mis, res, res_cs, res_co):
    """32-byte aligned output / bias / residual slices (every base pointer here is a fresh allocation; `bias_mis`: the bias pointer is
    16 bytes past a 32-byte boundary)"""
    return int(out_cs % 8 == 0 and out_co % 8 == 0 and not bias_mis and (res == "none" or (res_cs % 8 == 0 and res_co % 8 == 0)))


def row64_eligible(f16, passes, KH, KW, stride, pad, dil, cin_pad, BN, n_tiles, L, res_up, out_lo):
    return bool(f16 and passes == 3 and KH == 3 and KW == 3 and stride == 1 and pad == 1 and dil == 1 and cin_pad == 64 and BN <= 64
                and n_tiles == 1 and L == 1 and not res_up and not out_lo)


def out_hw(H, W, KH, KW, stride, pad, dil):
    return (H + 2 * pad - dil * (KH - 1) - 1) // stride + 1, (W + 2 * pad - dil * (KW - 1) - 1) // stride + 1


def env_of(c):
    return dict(c.env)


def launch_path(f16, passes, B, hws_out, Cin, Cout, KH, KW, stride, pad, dil, bn, v8, env, res_up=False, out_lo=False, L=1):
    """everything conv2d_tc_launch decides for a launch, as a dict"""
    bk = 64 if f16 else 32
    cin_pad = cdiv(Cin, bk) * bk
    m_tiles = sum(cdiv(Wo, TC_TW) * cdiv(Ho, TC_TH) * B for Ho, Wo in hws_out)
    if bn <= 0:
        BN = pick_bn_cost(Cout, m_tiles) if (f16 and passes in (2, 3)) else pick_bn_tf32(Cout)
    else:
        BN = bn
    BN = fit_bn(BN)
    n_tiles = cdiv(cdiv(Cout, 16) * 16, BN)
    row64 = row64_eligible(f16, passes, KH, KW, stride, pad, dil, cin_pad, BN, n_tiles, L, res_up, out_lo) and \
        str(env.get("VD3D_ROW64", "1")) != "0"
    stages, in_ring, split = ring_layout(BN, env.get("VD3D_TC_TILE_IN_RING"))
    chunk = max(1, int(env.get("VD3D_TC_CHUNK", 4)))
    return dict(BN=BN, n_tiles=n_tiles, m_tiles=m_tiles, cin_pad=cin_pad, KB=KH * KW * cin_pad // bk, chunk=chunk, row64=row64,
                stages=stages, staging="split" if split else "ring" if in_ring else "sep", v8=v8,
                mblock=mblock(m_tiles, n_tiles, stride, cin_pad, f16), epi_warps=tcp_epi_warps(BN), L=L)


def path_name(p):
    if p["row64"]:
        s = f"BN={p['BN']} v8={p['v8']} row64"
    else:
        s = f"BN={p['BN']} {p['staging']} v8={p['v8']}"
    if p["mblock"]:
        s += f" mblock={p['mblock']}"
    if p["L"] > 1:
        s += f" L={p['L']}"
    return s


# ---------------------------------------------------------------------------------------------------------------------------------------
# vd3d_conv2d_tc16, one level
# ---------------------------------------------------------------------------------------------------------------------------------------
# res: "none", "f32", "planes" (fp16 (hi, lo) residual planes) or "up" (fp32 residual at half the output size, read nearest-upsampled);
# outf: "f32", "planes" or "both".  The residual slice has the output's pitch and offset.  env: the engine's switches for the row.
Conv = namedtuple("Conv", "name B Cin in_cs in_co H W Cout out_cs out_co KH KW stride pad dil bn res outf relu bias_mis env reach")

CONV_CASES = [
    # 64-channel 3x3 convs (row-strip kernel): Cout % 8 == 4 tail in a 16-column tile, M = 1, M % 128 == 1 with Ho below the tile,
    # Cin 8 / 56 at a channel offset, and a v8 pair (out_co 4 / 8) on the same conv
    Conv("row64_bn16_tail12", 2, 64, 80, 8, 9, 17, 12, 20, 4, 3, 3, 1, 1, 1, 0, "f32", "both", True, False, (), "BN=16 v8=0 row64"),
    Conv("row64_m1_cout20", 1, 16, 24, 8, 1, 1, 20, 28, 4, 3, 3, 1, 1, 1, 0, "f32", "both", True, False, (), "BN=32 v8=0 row64"),
    Conv("row64_m129_planes", 1, 64, 64, 0, 3, 43, 64, 64, 0, 3, 3, 1, 1, 1, 0, "planes", "planes", False, True, (), "BN=64 v8=0 row64"),
    Conv("row64_cin8", 1, 8, 24, 8, 8, 16, 64, 64, 0, 3, 3, 1, 1, 1, 0, "none", "f32", True, False, (), "BN=64 v8=1 row64"),
    Conv("row64_cin56_v8off", 2, 56, 64, 8, 12, 20, 36, 40, 4, 3, 3, 1, 1, 1, 0, "f32", "both", True, False, (), "BN=48 v8=0 row64"),
    Conv("row64_cin56_v8on", 2, 56, 64, 8, 12, 20, 36, 48, 8, 3, 3, 1, 1, 1, 0, "f32", "both", True, False, (), "BN=48 v8=1 row64"),
    # conv2d_tcp_kernel
    Conv("bn32_5x5_pad3", 1, 16, 32, 8, 15, 17, 32, 40, 8, 5, 5, 1, 3, 1, 0, "none", "f32", False, False, (), "BN=32 sep v8=1"),
    Conv("bn48_1x7_kb7", 1, 40, 64, 24, 6, 21, 44, 52, 4, 1, 7, 1, 3, 1, 0, "planes", "both", True, True, (), "BN=48 ring v8=0"),
    Conv("bn64_7x1_s2_chunk1", 2, 56, 64, 8, 19, 10, 56, 64, 8, 7, 1, 2, 3, 1, 0, "f32", "planes", False, False,
         (("VD3D_TC_CHUNK", "1"),), "BN=64 ring v8=1"),
    Conv("bn80_req144_up", 1, 72, 96, 24, 12, 20, 132, 140, 4, 3, 3, 1, 1, 1, 144, "up", "both", True, False, (), "BN=80 ring v8=0"),
    Conv("bn80_policy_1x1", 1, 64, 64, 0, 9, 17, 80, 84, 4, 1, 1, 1, 0, 1, 0, "f32", "both", True, False, (), "BN=80 ring v8=0"),
    Conv("bn96_req192_s3_sep", 1, 136, 160, 24, 20, 23, 192, 200, 8, 3, 3, 3, 0, 1, 192, "f32", "f32", False, False,
         (("VD3D_TC_TILE_IN_RING", "0"),), "BN=96 sep v8=1"),
    Conv("bn96_policy_3x3", 1, 64, 72, 8, 10, 18, 96, 96, 0, 3, 3, 1, 1, 1, 0, "planes", "planes", True, False, (), "BN=96 ring v8=1"),
    Conv("bn112_s4_pad2", 2, 8, 16, 8, 33, 65, 104, 112, 4, 3, 3, 4, 2, 1, 0, "planes", "both", True, False, (), "BN=112 split v8=0"),
    Conv("bn128_req256_s2_d3_chunk64", 1, 64, 72, 8, 21, 25, 256, 264, 8, 3, 3, 2, 3, 3, 256, "none", "both", False, False,
         (("VD3D_TC_CHUNK", "64"),), "BN=128 split v8=1"),
    Conv("bn128_1x1_s2_sep", 1, 64, 64, 0, 17, 33, 128, 132, 4, 1, 1, 2, 0, 1, 0, "none", "both", True, False,
         (("VD3D_TC_TILE_IN_RING", "0"),), "BN=128 sep v8=0"),
    Conv("bn64_units180_kb1", 2, 8, 8, 0, 48, 48, 320, 320, 0, 1, 1, 1, 0, 1, 64, "f32", "f32", True, False, (), "BN=64 ring v8=1"),
    Conv("bn32_m255_d2_chunk1", 1, 40, 48, 8, 15, 17, 28, 32, 4, 3, 3, 1, 2, 2, 0, "none", "both", True, False,
         (("VD3D_TC_CHUNK", "1"),), "BN=32 sep v8=0"),
    Conv("bn16_1x3_d3_up_kb3", 1, 16, 40, 24, 10, 30, 16, 16, 0, 1, 3, 1, 3, 3, 0, "up", "f32", False, False, (), "BN=16 ring v8=1"),
    Conv("bn48_3x1_d2_s2", 2, 8, 16, 0, 17, 9, 48, 56, 8, 3, 1, 2, 1, 2, 0, "planes", "both", True, True, (), "BN=48 ring v8=0"),
    Conv("bn128_mblock_s4", 2, 136, 144, 8, 66, 130, 160, 168, 8, 3, 3, 4, 1, 1, 128, "f32", "f32", True, False, (),
         "BN=128 split v8=1 mblock=9"),
    Conv("bn16_req16_cout40", 1, 72, 80, 8, 7, 9, 40, 44, 4, 3, 3, 1, 1, 1, 16, "f32", "both", False, False,
         (("VD3D_TC_TILE_IN_RING", "1"),), "BN=16 ring v8=0"),
    Conv("bn112_req112_ring0", 1, 64, 64, 0, 9, 19, 108, 112, 0, 3, 3, 1, 2, 2, 112, "none", "f32", True, False,
         (("VD3D_TC_TILE_IN_RING", "0"),), "BN=112 sep v8=1"),
]


def conv_path(c, passes=3, env_override=None):
    env = env_of(c)
    if env_override:
        env.update(env_override)
    Ho, Wo = out_hw(c.H, c.W, c.KH, c.KW, c.stride, c.pad, c.dil)
    v8 = v8_ok(c.out_cs, c.out_co, c.bias_mis, c.res, c.out_cs, c.out_co)
    return launch_path(True, passes, c.B, [(Ho, Wo)], c.Cin, c.Cout, c.KH, c.KW, c.stride, c.pad, c.dil, c.bn, v8, env,
                       res_up=c.res == "up")


# ---------------------------------------------------------------------------------------------------------------------------------------
# vd3d_conv2d_tc16, multi-level launches (L = 2 .. TC_MAX_LEVELS); every level has the same channel layout, its own input tensor, and its
# outputs (residual) at a pixel offset inside one allocation per form, GAP sentinel pixels after the previous level
# ---------------------------------------------------------------------------------------------------------------------------------------
Multi = namedtuple("Multi", "name B Cin in_cs in_co hws Cout out_cs out_co KH KW stride pad bn res outf relu reach")
LEVEL_GAP = 5

MULTI_CASES = [
    Multi("L2_up", 1, 64, 64, 0, ((16, 32), (8, 16)), 64, 64, 0, 3, 3, 1, 1, 0, "up", "both", True, "BN=64 ring v8=1 L=2"),
    Multi("L3_1x1_level", 1, 40, 48, 8, ((13, 27), (7, 14), (1, 1)), 44, 52, 4, 3, 3, 1, 1, 0, "f32", "planes", False, "BN=48 ring v8=0 L=3"),
    Multi("L4_s2_ragged", 1, 72, 96, 24, ((24, 40), (12, 20), (6, 10), (2, 2)), 100, 104, 0, 3, 3, 2, 1, 0, "f32", "both", True,
          "BN=112 split v8=1 L=4"),
    Multi("L5_up", 1, 64, 64, 0, ((32, 64), (16, 32), (8, 16), (4, 8), (2, 4)), 96, 96, 0, 3, 3, 1, 1, 0, "up", "both", True,
          "BN=96 ring v8=1 L=5"),
    Multi("L5_1x1_units", 2, 16, 32, 8, ((40, 80), (20, 40), (10, 20), (5, 10), (1, 1)), 256, 264, 8, 1, 1, 1, 0, 128, "none", "f32", False,
          "BN=128 split v8=1 L=5"),
]


def multi_out_hws(c):
    return [out_hw(H, W, c.KH, c.KW, c.stride, c.pad, 1) for H, W in c.hws]


def multi_path(c):
    v8 = v8_ok(c.out_cs, c.out_co, False, c.res, c.out_cs, c.out_co)
    return launch_path(True, 3, c.B, multi_out_hws(c), c.Cin, c.Cout, c.KH, c.KW, c.stride, c.pad, 1, c.bn, v8, {},
                       res_up=c.res == "up", L=len(c.hws))


def level_offsets(B, hws):
    """pixel offset of every level inside one allocation (LEVEL_GAP sentinel pixels between levels), and the allocation's pixel count with
    one more image of the last level after it"""
    offs, p = [], 0
    for Ho, Wo in hws:
        offs.append(p)
        p += B * Ho * Wo + LEVEL_GAP
    return offs, p + hws[-1][0] * hws[-1][1]


# ---------------------------------------------------------------------------------------------------------------------------------------
# vd3d_convtranspose2d_tc16: ConvTranspose2d(4, stride 2, pad 1) as four phase levels over one input
# ---------------------------------------------------------------------------------------------------------------------------------------
ConvT = namedtuple("ConvT", "name B Cin in_cs in_co H W Cout out_cs out_co bn outf relu reach")

CONVT_CASES = [
    ConvT("h1_w1", 1, 8, 16, 8, 1, 1, 16, 16, 0, 0, "both", True, "BN=16 ring v8=1 L=4"),
    ConvT("odd_planes_only", 2, 40, 64, 24, 5, 7, 48, 56, 4, 0, "planes", False, "BN=48 ring v8=0 L=4"),
    ConvT("w1_cout144_picker", 1, 72, 80, 8, 3, 1, 144, 152, 8, 0, "both", True, "BN=64 ring v8=1 L=4"),
    ConvT("cout208_picker", 1, 64, 64, 0, 9, 13, 208, 212, 4, 0, "f32", True, "BN=64 ring v8=0 L=4"),
    ConvT("bn128_cout256", 1, 16, 24, 8, 6, 10, 256, 256, 0, 128, "both", False, "BN=128 split v8=1 L=4"),
]


def convt_path(c):
    v8 = v8_ok(c.out_cs, c.out_co, False, "none", 0, 0)
    return launch_path(True, 3, c.B, [(c.H, c.W)] * 4, c.Cin, c.Cout, 2, 2, 1, 1, 1, c.bn, v8, {}, L=4)


# ---------------------------------------------------------------------------------------------------------------------------------------
# vd3d_conv2d_tc (3xTF32, stride 1): passes 1 and 3, the tf32 `lo` companion output
# ---------------------------------------------------------------------------------------------------------------------------------------
Tf32 = namedtuple("Tf32", "name B Cin in_cs in_co H W Cout out_cs out_co K pad dil bn res out_lo relu passes reach")

TF32_CASES = [
    Tf32("p1_bn16_1x1", 1, 32, 32, 0, 8, 16, 16, 16, 0, 1, 0, 1, 0, False, False, False, 1, "BN=16 ring v8=1"),
    Tf32("p3_bn96_lo", 1, 64, 96, 32, 9, 20, 96, 104, 8, 3, 1, 1, 0, True, True, True, 3, "BN=96 ring v8=1"),
    Tf32("p3_bn48_d2", 1, 32, 40, 8, 7, 11, 144, 148, 4, 3, 2, 2, 0, False, True, False, 3, "BN=48 ring v8=0"),
    Tf32("p3_bn128_ragged", 1, 32, 32, 0, 6, 13, 200, 208, 8, 1, 0, 1, 0, True, False, True, 3, "BN=128 split v8=1"),
    Tf32("p1_req64", 2, 64, 64, 0, 5, 9, 36, 40, 4, 3, 1, 1, 64, False, True, True, 1, "BN=64 ring v8=0"),
]


def tf32_path(c):
    v8 = v8_ok(c.out_cs, c.out_co, False, "f32" if c.res else "none", c.out_cs, c.out_co)
    Ho, Wo = out_hw(c.H, c.W, c.K, c.K, 1, c.pad, c.dil)
    return launch_path(False, c.passes, c.B, [(Ho, Wo)], c.Cin, c.Cout, c.K, c.K, 1, c.pad, c.dil, c.bn, v8, {}, out_lo=c.out_lo)


# ---------------------------------------------------------------------------------------------------------------------------------------
# operands
# ---------------------------------------------------------------------------------------------------------------------------------------
EXACT_X, EXACT_W8, EXACT_B8, EXACT_R = 4, 8, 16, 8           # |x| <= 4, |8 w| <= 8, |8 b| <= 16, |r| <= 8


def exact_operands(B, Cin, H, W, Cout, KH, KW, res_shape, seed, w_layout="conv"):
    """x [B, Cin, H, W] integers, w multiples of 1/8 with max |w| = 1 exactly ([Cout, Cin, KH, KW], or [Cin, Cout, KH, KW] for a transposed
    conv), bias [Cout] multiples of 1/8, residual integers of res_shape (or None); all float64"""
    g = torch.Generator().manual_seed(seed)
    ri = lambda lim, *s: torch.randint(-lim, lim + 1, s, generator=g).double()
    x = ri(EXACT_X, B, Cin, H, W)
    wshape = (Cout, Cin, KH, KW) if w_layout == "conv" else (Cin, Cout, KH, KW)
    w = ri(EXACT_W8, *wshape) / 8
    w.view(-1)[0] = 1.0
    b = ri(EXACT_B8, Cout) / 8
    r = ri(EXACT_R, *res_shape) if res_shape is not None else None
    return x, w, b, r


def exact_grid_limit(K):
    """largest |partial sum| of the exact operands in units of 1/8 (the grid every product and sum lies on): K products of |x| <= 4 and
    |w| <= 1, then the residual and the bias"""
    return 8 * (K * EXACT_X * 1 + EXACT_R + EXACT_B8 / 8)


def normal_operands(B, Cin, H, W, Cout, KH, KW, res_shape, seed, wscale=1.0, w_layout="conv"):
    """x float32 normals (as float64), w float64 normals / sqrt(fan-in) * wscale, bias and residual float32 normals"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Cin, H, W, generator=g).double()
    wshape = (Cout, Cin, KH, KW) if w_layout == "conv" else (Cin, Cout, KH, KW)
    w = torch.randn(*wshape, generator=g, dtype=torch.float64) / math.sqrt(Cin * KH * KW) * wscale
    b = torch.randn(Cout, generator=g).double()
    r = torch.randn(*res_shape, generator=g).double() if res_shape is not None else None
    return x, w, b, r


def split16(v):
    """float64 / float32 tensor -> (hi, lo) fp16 with hi = rn16(v), lo = rn16(v - hi), v taken in float32 (as split_h16_kernel)"""
    v = v.float()
    hi = v.half()
    return hi, (v - hi.float()).half()


def pack_weight(w, cin64):
    """[Cout, Cin, KH, KW] float64 -> [Cout][KH*KW*cin64] with k = tap * cin64 + ci (ConvLayer's packing)"""
    Cout, Cin, KH, KW = w.shape
    wk = torch.zeros(Cout, KH * KW, cin64, dtype=torch.float64)
    wk[:, :, :Cin] = w.permute(0, 2, 3, 1).reshape(Cout, KH * KW, Cin)
    return wk.reshape(Cout, KH * KW * cin64)


# ---------------------------------------------------------------------------------------------------------------------------------------
# float64 references
# ---------------------------------------------------------------------------------------------------------------------------------------
def up2(r):
    return r.repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)


def conv_ref(x, w, b, r, stride, pad, dil, relu, res_up=False):
    """float64 conv folded as the epilogue orders it: acc * out_scale + residual, then + bias, then ReLU.  Also returns the magnitude sums
    the bound takes: S = conv(|x|, |w|), SW = conv(1, |w|) over the in-image taps, SX = conv(|x|, 1)."""
    acc = F.conv2d(x, w, None, stride=stride, padding=pad, dilation=dil)
    S = F.conv2d(x.abs(), w.abs(), None, stride=stride, padding=pad, dilation=dil)
    SW = F.conv2d(torch.ones_like(x), w.abs(), None, stride=stride, padding=pad, dilation=dil)
    SX = F.conv2d(x.abs(), torch.ones_like(w), None, stride=stride, padding=pad, dilation=dil)
    return epilogue_ref(acc, b, r, relu, res_up), (S, SW, SX)


def epilogue_ref(acc, b, r, relu, res_up=False):
    out = acc
    if r is not None:
        out = out + (up2(r) if res_up else r)
    out = out + b.view(1, -1, 1, 1)
    return out.clamp_min(0) if relu else out


def convt_ref(x, wt, b, relu):
    """ConvTranspose2d(4, stride 2, pad 1) in float64 (not through the phase packing); magnitude sums as conv_ref"""
    acc = F.conv_transpose2d(x, wt, None, stride=2, padding=1)
    S = F.conv_transpose2d(x.abs(), wt.abs(), None, stride=2, padding=1)
    SW = F.conv_transpose2d(torch.ones_like(x), wt.abs(), None, stride=2, padding=1)
    SX = F.conv_transpose2d(x.abs(), torch.ones_like(wt), None, stride=2, padding=1)
    return epilogue_ref(acc, b, None, relu), (S, SW, SX)


# ---------------------------------------------------------------------------------------------------------------------------------------
# per-element error bounds of random-normal operands
# ---------------------------------------------------------------------------------------------------------------------------------------
# fp16 split of an activation x (hi = rn16(x), lo = rn16(x - hi)): |x - hi - lo| <= 2^-22 |x| (+ 2^-25 when lo, or hi, is subnormal).  A
# weight w is first scaled by S = 2^k and rounded to float32 (2^-24), then split the same way; the subnormal term is 2^-25 / S = 2^-25 out_scale
# (the clamp of k at 2^+-24 leaves small weights with subnormal planes).  The engine drops x_lo w_lo: |x_lo| |w_lo| <= 2^-22 |x| |w| (1 + 2^-9).
SPLIT16 = 2.0 ** -22 * (2.0 + 2.0 ** -2) * (1 + 2.0 ** -9)
DROP16 = 2.0 ** -22 * (1 + 2.0 ** -9)
SUB16 = 2.0 ** -25 * 2
# 3xTF32: the MMA reads the top 19 bits, so hi and trunc13(lo) carry x to within 2^-20 |x| (same for w); the dropped lo * lo < 2^-20 |x| |w|.
# One pass reads only trunc13(x) and trunc13(w): 2^-10 each.
SPLIT_TF32 = {3: 3 * 2.0 ** -20 + 2.0 ** -24, 1: 2.0 ** -9 + 2.0 ** -20 + 2.0 ** -24}
# tensor-core accumulation: within a promotion chunk every MMA instruction adds its products to the running fp32 sum with truncation, at most
# one unit in the last place of the running magnitude (2^-23 |running|); the chunks are added to the total with round-to-nearest (2^-24 each);
# the epilogue rounds acc * out_scale + residual and then + bias (2^-24 each, out_scale is a power of two).
TRUNC = 2.0 ** -23
RN = 2.0 ** -24


def mma_per_kblock(f16, passes):
    """MMA instructions per k-block: 128-byte operand rows = 4 K steps (16 fp16 / 8 tf32 elements), each one MMA per product"""
    return 4 * (3 if passes in (2, 3) else 1)


def accumulation_factor(KB, chunk, f16=True, passes=3):
    """relative bound (over sum |x| |w|) of the chunked truncating accumulation and the round-to-nearest promotions"""
    n_mma = mma_per_kblock(f16, passes) * min(chunk, KB)
    n_chunks = cdiv(KB, chunk)
    return (TRUNC * n_mma + RN * n_chunks) * (1 + 2.0 ** -9)


def tc16_bound(mags, KB, chunk, out_scale, r, b, res_up=False, res_planes=False):
    """per-element bound of |device - float64| for the fp16-split engine with float64 weights w (out_scale = 1 / the weight scale); `mags` =
    (S, SW, SX) of conv_ref"""
    S, SW, SX = mags
    bound = S * (SPLIT16 + DROP16 + accumulation_factor(KB, chunk)) + SUB16 * (SW + out_scale * SX)
    ra = torch.zeros_like(S) if r is None else (up2(r) if res_up else r).abs()
    bound = bound + 2 * RN * (S * (1 + 2.0 ** -9) + ra + b.abs().view(1, -1, 1, 1))
    if res_planes:
        bound = bound + 2.0 ** -22 * ra + SUB16
    return bound


def tf32_bound(mags, KB, chunk, passes, r, b):
    S, _, _ = mags
    ra = torch.zeros_like(S) if r is None else r.abs()
    return S * (SPLIT_TF32[passes] + accumulation_factor(KB, chunk, False, passes)) + \
        2 * RN * (S * (1 + 2.0 ** -8) + ra + b.abs().view(1, -1, 1, 1))


def planes_bound(want, bound):
    """extra error of a value read back from its own fp16 (hi, lo) planes"""
    return 2.0 ** -22 * (want.abs() + bound) + SUB16


def err_ratio(got, want, bound):
    """max |got - want| / bound (an element with zero error counts 0; a non-finite result is inf)"""
    err = (got.double() - want.double()).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bound.double())
    r = torch.where(torch.isfinite(got.double()), r, torch.full_like(r, math.inf))
    return float(r.max()) if r.numel() else 0.0


# ---------------------------------------------------------------------------------------------------------------------------------------
# host restatement of the engine's arithmetic, for the CPU checks that the comparisons catch known-wrong kernels
# ---------------------------------------------------------------------------------------------------------------------------------------
def plane_conv(xh, xl, wh, wl, osc, stride, pad, dil, products=("lo_hi", "hi_lo", "hi_hi")):
    """float64 sum of the chosen plane products (exact products, exact sums), times out_scale: the engine's value before its roundings.
    passes = 2 drops "lo_hi" (A_lo * W_hi)."""
    terms = {"lo_hi": (xl, wh), "hi_lo": (xh, wl), "hi_hi": (xh, wh), "lo_lo": (xl, wl)}
    acc = 0
    for p in products:
        a, w = terms[p]
        acc = acc + F.conv2d(a.double(), w.double(), None, stride=stride, padding=pad, dilation=dil)
    return acc * osc


def epilogue_f32(acc, b, r, relu, residual_first=True):
    """the epilogue in float32: (acc + r) + b as the engine does, or (acc + b) + r"""
    a, bb = acc.float(), b.float().view(1, -1, 1, 1)
    rr = torch.zeros_like(a) if r is None else r.float()
    out = (a + rr) + bb if residual_first else (a + bb) + rr
    return out.clamp_min(0) if relu else out
