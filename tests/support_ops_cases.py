"""Constructed cases for the fp32 support kernels, their float64 references and restatements of the host-side selection logic.

Kernels: the SIMT implicit-GEMM conv (csrc/conv2d_simt.cu), the NCHW <-> NHWC converters, max / average pools, depthwise 3x3 conv,
channel copy and the DLA depthwise transposed conv (csrc/pool_misc.cu), LookGround's sampler (csrc/look_ground.cu) and the fp16 / tf32
splitters at the end of csrc/conv2d_tc.cu.

Two kinds of operands are used:
  * exact: small integers and dyadic fractions (multiples of 1/8) chosen so that every product and every partial sum is representable in
    float32.  Whatever order a kernel accumulates in, it must then equal the float64 reference bit for bit, so a wrong tap, pixel, channel or
    border shows up as a plain inequality;
  * normal: random normals, compared with a per-element forward-error bound.  A sequential float32 chain of n roundings (fma or add) over
    terms whose magnitudes sum to S is within gamma(n) * S of the exact sum, gamma(n) = n u / (1 - n u), u = 2^-24 (Higham, Accuracy and
    Stability of Numerical Algorithms, 3.1).  S is computed by the same float64 operation on |operands|.

Every device run writes into a channel slice of a wider buffer filled with SENTINEL and reads its input from a slice whose neighbouring
channels hold SENTINEL too, so reading or writing the wrong channel changes the result.
"""
from collections import namedtuple

import torch
import torch.nn.functional as F

U = 2.0 ** -24
SENTINEL = -777.25                        # finite, exact, and far outside every operand range used here


def gamma(n):
    return n * U / (1.0 - n * U)


def err_ratio(got, want, bound):
    """max |got - want| / bound; an element with a zero bound must be exact (its ratio is 0 if equal, inf otherwise)"""
    err = (got.double() - want.double()).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bound.double())
    return float(r.max()) if r.numel() else 0.0


# ---------------------------------------------------------------------------------------------------------------------------------------
# SIMT conv (vd3d_conv2d_nhwc)
# ---------------------------------------------------------------------------------------------------------------------------------------
CBM, CBK = 128, 16                        # the kernel's CTA tile rows and K chunk


def simt_select(Cin, in_cs, in_co, Cout, aligned=True):
    """(BN, VEC) of the instantiation vd3d_conv2d_nhwc launches: the float4 gather needs Cin, the input pitch and offset to be multiples of 4
    and a 16-byte aligned base pointer; the column tile is the smallest of 128 / 64 / 32 / 16 that the thresholds 64 / 32 / 16 allow."""
    vec = 4 if (Cin % 4 == 0 and in_cs % 4 == 0 and in_co % 4 == 0 and aligned) else 1
    bn = 128 if Cout > 64 else 64 if Cout > 32 else 32 if Cout > 16 else 16
    return bn, vec


def out_hw(H, W, KH, KW, stride, pad, dil):
    return (H + 2 * pad - dil * (KH - 1) - 1) // stride + 1, (W + 2 * pad - dil * (KW - 1) - 1) // stride + 1


ConvCase = namedtuple("ConvCase", "name B Cin H W Cout KH KW stride pad dil bias res relu in_cs in_co reach")

# reach = (BN, VEC); TN = BN / 16 columns per thread: TN = 1, 2 store scalars, TN = 4, 8 store float4
CONV_CASES = [
    ConvCase("k3_bn16_scalar", 2, 3, 7, 9, 4, 1, 1, 1, 0, 1, True, False, False, 5, 1, (16, 1)),           # K = 3, Cout = 4, TN = 1
    ConvCase("m129_bn16_vec", 1, 4, 3, 43, 16, 1, 1, 1, 0, 1, False, False, True, 12, 4, (16, 4)),          # M % 128 = 1, K = 4
    ConvCase("bn16_scalar_cout16", 1, 12, 6, 5, 16, 3, 3, 1, 1, 1, True, True, False, 16, 2, (16, 1)),    # in_co = 2 -> scalar, K = 108
    ConvCase("bn32_scalar_s2", 2, 6, 9, 11, 20, 3, 3, 2, 1, 1, True, False, True, 10, 2, (32, 1)),         # Cout = 20, TN = 2, stride 2
    ConvCase("bn32_vec_1x7", 1, 12, 5, 19, 32, 1, 7, 1, 3, 1, False, True, False, 16, 4, (32, 4)),         # 1x7, K = 84 (% 16 = 4)
    ConvCase("bn64_scalar_7x1_d2", 1, 5, 13, 6, 36, 7, 1, 1, 3, 2, True, False, True, 5, 0, (64, 1)),      # 7x1, dilation 2, Cout = 36
    ConvCase("bn64_vec_m255", 1, 28, 15, 17, 64, 3, 3, 1, 1, 1, True, True, True, 32, 4, (64, 4)),         # M % 128 = 127, K = 252 (% 16 = 12)
    ConvCase("bn64_scalar_tiny_in", 1, 3, 2, 3, 64, 7, 7, 2, 3, 1, False, False, True, 3, 0, (64, 1)),     # 2x3 input under a 13x13 footprint
    ConvCase("bn128_scalar_3x1_s3d3", 2, 8, 17, 10, 68, 3, 1, 3, 4, 3, True, True, False, 12, 2, (128, 1)),  # Cout = 68, 3x1, stride 3, dil 3, pad 4 > k/2
    ConvCase("bn128_vec_s3_p0", 1, 16, 20, 23, 128, 3, 3, 3, 0, 1, True, True, True, 24, 8, (128, 4)),     # stride 3, pad 0
    ConvCase("bn128_vec_cout132_d3", 1, 32, 9, 11, 132, 3, 3, 1, 3, 3, True, False, False, 40, 4, (128, 4)),  # ragged second column tile
    ConvCase("bn128_scalar_cout260", 1, 7, 9, 8, 260, 5, 5, 2, 4, 1, False, True, True, 9, 1, (128, 1)),   # three column tiles, pad 4 > k/2
    ConvCase("m1_bn16_vec", 1, 8, 1, 1, 16, 3, 3, 1, 1, 1, True, False, True, 8, 0, (16, 4)),              # M = 1
    ConvCase("bn32_vec_k12", 2, 4, 7, 6, 24, 1, 3, 1, 1, 1, True, False, False, 4, 0, (32, 4)),            # K = 12
    ConvCase("bn128_scalar_k_tail", 1, 20, 6, 7, 128, 3, 3, 1, 1, 2, True, False, True, 24, 2, (128, 1)),  # K = 180 (% 16 = 4), dilation 2
]

# same conv, in_co = 4 (float4 gather) versus in_co = 2 (scalar gather) on identical data: both fill As[k][m] with the same value in the same
# k order, so the outputs must be identical bit for bit.  One row per column tile.
# name, B, Cin, H, W, Cout, KH, KW, stride, pad, dil, in_cs
PAIR_CASES = [
    ("pair_bn16", 2, 8, 9, 13, 16, 3, 3, 1, 1, 1, 16),
    ("pair_bn32", 1, 12, 11, 14, 32, 3, 3, 2, 2, 1, 20),
    ("pair_bn64", 1, 16, 12, 9, 64, 1, 5, 1, 2, 2, 24),
    ("pair_bn128", 1, 20, 10, 12, 132, 3, 3, 1, 1, 1, 28),
]
PAIR_IN_CO = (4, 2)


def conv_dims(c):
    Ho, Wo = out_hw(c.H, c.W, c.KH, c.KW, c.stride, c.pad, c.dil)
    return Ho, Wo, c.B * Ho * Wo, c.KH * c.KW * c.Cin


def conv_operands(c, kind, seed):
    """x [B, Cin, H, W], w [Cout, Cin, KH, KW], b [Cout] or None, r [B, Cout, Ho, Wo] or None, all float32.
    exact: x in [-4, 4], w and b multiples of 1/8 in [-1, 1] and [-2, 2], r in [-8, 8]."""
    g = torch.Generator().manual_seed(seed)
    Ho, Wo, _, K = conv_dims(c)
    ri = lambda lo, hi, *s: torch.randint(lo, hi + 1, s, generator=g).float()
    if kind == "exact":
        x = ri(-4, 4, c.B, c.Cin, c.H, c.W)
        w = ri(-8, 8, c.Cout, c.Cin, c.KH, c.KW) / 8
        b = ri(-16, 16, c.Cout) / 8 if c.bias else None
        r = ri(-8, 8, c.B, c.Cout, Ho, Wo) if c.res else None
    else:
        x = torch.randn(c.B, c.Cin, c.H, c.W, generator=g)
        w = torch.randn(c.Cout, c.Cin, c.KH, c.KW, generator=g) / K ** 0.5
        b = torch.randn(c.Cout, generator=g) if c.bias else None
        r = torch.randn(c.B, c.Cout, Ho, Wo, generator=g) if c.res else None
    return x, w, b, r


def exact_sum_limit(c):
    """Largest |partial sum| the exact operands can reach: K * 4 * 1 + 2 + 8.  All partial sums are multiples of 1/8, so they are exact in
    float32 while this stays below 2^21."""
    return conv_dims(c)[3] * 4 + 2 + 8


def pack_conv_weight(w):
    """[Cout, Cin, KH, KW] -> the kernel's [K, Cout] with k = (kh * KW + kw) * Cin + ci."""
    return w.permute(2, 3, 1, 0).reshape(-1, w.shape[0]).contiguous()


def conv_ref(x, w, b, r, stride, pad, dil, relu):
    """float64 conv (+ bias) (+ residual) (+ ReLU) and S = the same conv on |x|, |w| + |b| + |r|; both [B, Cout, Ho, Wo]."""
    x, w = x.double(), w.double()
    out = F.conv2d(x, w, None if b is None else b.double(), stride=stride, padding=pad, dilation=dil)
    S = F.conv2d(x.abs(), w.abs(), None if b is None else b.double().abs(), stride=stride, padding=pad, dilation=dil)
    if r is not None:
        out, S = out + r.double(), S + r.double().abs()
    if relu:
        out = out.clamp_min(0)
    return out, S


# ---------------------------------------------------------------------------------------------------------------------------------------
# layout converters
# ---------------------------------------------------------------------------------------------------------------------------------------
def nchw_to_nhwc_kernel(C):
    """the kernel vd3d_nchw_to_nhwc launches: one thread per pixel for C <= 4, the 32 x 32 shared-memory transpose otherwise"""
    return "small" if C <= 4 else "tiled"


LAYOUT_C = (1, 3, 4, 5, 31, 33, 64)
LAYOUT_HW = ((3, 5), (7, 9), (4, 16))            # HW = 15 < 32, 63 (% 32 != 0), 64
LAYOUT_CO = 3                                    # channel offset of the NHWC side; its pitch is C + 5


# ---------------------------------------------------------------------------------------------------------------------------------------
# pools, depthwise convs, channel copy
# ---------------------------------------------------------------------------------------------------------------------------------------
MAXPOOL3_HW = ((1, 1), (1, 2), (2, 3), (3, 1), (3, 6), (7, 7), (6, 8), (9, 4))
MAXPOOL2_HW = ((2, 2), (3, 3), (5, 7), (7, 4), (2, 9))
AVGPOOL_HW = ((2, 2), (4, 6), (8, 10))
POOL_KINDS = ("normal", "negative", "inf")       # negative: every value < 0, so a zero-padded window would show; inf: +-inf entries


def pool_input(B, C, H, W, kind, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, C, H, W, generator=g)
    if kind == "negative":
        x = -(x.abs() + 0.5)
    elif kind == "inf":
        pick = torch.rand(B, C, H, W, generator=g)
        x = torch.where(pick < 0.1, torch.full_like(x, float("inf")), torch.where(pick > 0.85, torch.full_like(x, float("-inf")), x))
    elif kind == "dyadic":
        x = torch.randint(-64, 65, (B, C, H, W), generator=g).float() / 16
    return x


def maxpool3_out_hw(H, W):
    return (H - 1) // 2 + 1, (W - 1) // 2 + 1


def maxpool3_ref(x):
    return F.max_pool2d(x.double(), 3, 2, 1)        # torch pads max pooling with -inf


def maxpool2_ref(x):
    return F.max_pool2d(x.double(), 2, 2)           # floor: the last row / column of an odd size is dropped


def avgpool2_ref(x):
    """float64 mean of each 2x2 window and S = sum |x| / 4: the kernel adds the four values in row-major order (3 roundings), then divides
    by 4 exactly."""
    x = x.double()
    return F.avg_pool2d(x, 2), F.avg_pool2d(x.abs(), 2)


# B, H, W, C, bias, relu
DWCONV_CASES = [(2, 1, 5, 4, False, False), (1, 6, 1, 8, True, True), (1, 1, 1, 4, True, False), (2, 5, 7, 132, True, True),
                (1, 4, 3, 132, False, True)]


def dwconv_operands(B, H, W, C, bias, kind, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "exact":
        x = torch.randint(-8, 9, (B, C, H, W), generator=g).float()
        w = torch.randint(-8, 9, (C, 1, 3, 3), generator=g).float() / 8
        b = torch.randint(-16, 17, (C,), generator=g).float() / 8 if bias else None
    else:
        x = torch.randn(B, C, H, W, generator=g)
        w = torch.randn(C, 1, 3, 3, generator=g) / 3
        b = torch.randn(C, generator=g) if bias else None
    return x, w, b


def dwconv_ref(x, w, b, relu):
    """float64 depthwise 3x3 / pad 1 (+ bias) (+ ReLU) and S; the kernel runs 9 fmas and one bias add: gamma(10)."""
    C = x.shape[1]
    out = F.conv2d(x.double(), w.double(), None if b is None else b.double(), padding=1, groups=C)
    S = F.conv2d(x.double().abs(), w.double().abs(), None if b is None else b.double().abs(), padding=1, groups=C)
    return (out.clamp_min(0) if relu else out), S


# B, H, W, C, f, addend
DWT_CASES = [(2, 3, 5, 4, 2, True), (1, 1, 7, 8, 2, False), (2, 3, 5, 4, 4, False), (1, 1, 1, 8, 4, True), (1, 5, 3, 4, 8, True),
             (2, 1, 3, 12, 8, False), (1, 2, 2, 4, 8, False)]


def dwt_operands(B, H, W, C, f, addend, kind, seed):
    g = torch.Generator().manual_seed(seed)
    K = 2 * f
    if kind == "exact":
        x = torch.randint(-8, 9, (B, C, H, W), generator=g).float()
        w = torch.randint(-8, 9, (C, 1, K, K), generator=g).float() / 8
        a = torch.randint(-8, 9, (B, C, H * f, W * f), generator=g).float() if addend else None
    else:
        x = torch.randn(B, C, H, W, generator=g)
        w = torch.randn(C, 1, K, K, generator=g) / 2
        a = torch.randn(B, C, H * f, W * f, generator=g) if addend else None
    return x, w, a


def dwt_ref(x, w, a, f):
    """float64 depthwise ConvTranspose2d(kernel 2f, stride f, padding f/2) (+ addend) and S.  Each output pixel takes at most 2 x 2 input
    pixels: 4 fmas and one add, gamma(5)."""
    C = x.shape[1]
    out = F.conv_transpose2d(x.double(), w.double(), None, stride=f, padding=f // 2, groups=C)
    S = F.conv_transpose2d(x.double().abs(), w.double().abs(), None, stride=f, padding=f // 2, groups=C)
    if a is not None:
        out, S = out + a.double(), S + a.double().abs()
    return out, S


def dwt_taps_per_output(H, W, f):
    """number of (iy, ix) input pixels that reach each output pixel: [H f, W f] int (the counting form of dw_convtranspose's loop)"""
    K, pad = 2 * f, f // 2
    y = torch.arange(H * f)
    x = torch.arange(W * f)
    ny = sum(((y + pad - iy * f >= 0) & (y + pad - iy * f < K)).long() for iy in range(H))
    nx = sum(((x + pad - ix * f >= 0) & (x + pad - ix * f < K)).long() for ix in range(W))
    return ny[:, None] * nx[None, :]


# npix (B, H, W), C, in_cs, in_co, out_cs, out_co
COPY_CASES = [((2, 5, 7), 24, 32, 4, 40, 8), ((1, 1, 1), 4, 4, 0, 12, 8), ((3, 9, 11), 132, 136, 4, 140, 0)]


# ---------------------------------------------------------------------------------------------------------------------------------------
# LookGround's sampler (vd3d_look_ground_sample)
# ---------------------------------------------------------------------------------------------------------------------------------------
LGCase = namedtuple("LGCase", "name B C H W x_cs x_co d_cs d_co elev cy_frac dconv")
# cy_frac: cy / 16 as a fraction of H - 1 (below 1: the rows under cy are shifted down, the last ones clamped to the bottom row);
# dconv: 'normal' learned offsets or 'zero' (tanh(0) = 0: no offset).
LG_CASES = [
    LGCase("bottom_c4", 2, 4, 12, 21, 12, 4, 4, 1, 1.65, 0.3, "normal"),       # rows past the bottom border, one channel quad
    LGCase("bottom_c132_wrap", 2, 132, 9, 14, 140, 4, 8, 3, 1.65, 0.25, "normal"),   # 132 channels: lane 0 takes quads 0 and 32
    LGCase("elev_other", 3, 8, 10, 17, 8, 0, 2, 0, 1.3, 0.5, "normal"),       # relative elevation other than 1.65
    LGCase("integer_grid", 2, 8, 9, 17, 16, 8, 3, 2, 1.65, 1.5, "zero"),     # H - 1, W - 1 powers of 2, no shift: every tap on an integer
    LGCase("integer_grid_c132", 1, 132, 5, 33, 136, 4, 1, 0, 1.5, 1.2, "zero"),
    LGCase("h2_w2", 2, 4, 2, 2, 8, 4, 4, 2, 1.65, 0.2, "normal"),
    LGCase("h2_w2_elev", 1, 12, 2, 2, 12, 0, 1, 0, 1.3, 0.0, "normal"),
]
LG_BASELINE = 0.54
LG_H_MEAN = 1.535


def lg_out_cs(c):
    return c.C + 4                               # C sampled channels, the disparity channel C and 3 channels the kernel must not touch


def lg_inputs(c, seed):
    """x [B, C, H, W], dconv [B, H, W] (the disp_create conv's output), P2 [B, 3, 4] (a different camera per image), all float32."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(c.B, c.C, c.H, c.W, generator=g)
    d = torch.randn(c.B, c.H, c.W, generator=g) * 2 if c.dconv == "normal" else torch.zeros(c.B, c.H, c.W)
    P2 = torch.zeros(c.B, 3, 4)
    for b in range(c.B):
        f = 700.0 + 15.0 * b
        P2[b, 0, 0], P2[b, 0, 2], P2[b, 0, 3] = f, 600.0 + 3 * b, 44.0 + b
        P2[b, 1, 1], P2[b, 1, 2], P2[b, 1, 3] = f, 16.0 * (c.cy_frac * (c.H - 1) + 0.37 * b * (c.cy_frac > 0)), 0.2 - 0.1 * b
        P2[b, 2, 2], P2[b, 2, 3] = 1.0, 0.003
    return x, d, P2


def lg_flow(dconv, P2, H, W, elev):
    """The sampling grid [B, H, W, 2] in float32, in torch_port.look_ground's op order (dconv = the disp_create conv's output)."""
    B = dconv.shape[0]
    P2 = P2.clone()
    P2[:, 0:2] /= 16.0
    disp = torch.tanh(dconv.float())
    disp = 0.1 * (0.05 * disp + 0.95 * disp)
    yy = torch.arange(H, dtype=torch.float32).view(1, H, 1).expand(1, H, W)
    cy = P2[:, 1:2, 2:3]
    x_base = torch.linspace(-1, 1, W).repeat(B, H, 1)
    y_base = torch.linspace(-1, 1, H).repeat(B, W, 1).transpose(1, 2)
    y_shifts_base = F.relu(LG_H_MEAN * (yy - cy) / (2 * (elev - 0.5 * LG_H_MEAN))) / (yy.shape[1] * 0.5)
    y_shifts = y_shifts_base + disp
    return torch.stack((x_base, y_base + y_shifts), dim=3)


def lg_disparity(P2, H, W, elev, baseline=LG_BASELINE):
    """the disparity plane [B, 1, H, W] in float32, in torch_port.look_ground's op order"""
    P2 = P2.clone()
    P2[:, 0:2] /= 16.0
    yy = torch.arange(H, dtype=torch.float32).view(1, H, 1).expand(1, H, W)
    fy, cy, Ty = P2[:, 1:2, 1:2], P2[:, 1:2, 2:3], P2[:, 1:2, 3:4]
    return F.relu(fy * baseline * (yy - cy) / (torch.abs(fy * elev + Ty) + 1e-10)).unsqueeze(1)


def lg_pixel_coords(flow, H, W):
    """grid_sample's unnormalisation (align_corners=True) and border clip, in float64: ix, iy [B, H, W]"""
    f = flow.double()
    ix = ((f[..., 0] + 1) / 2 * (W - 1)).clamp(0, W - 1)
    iy = ((f[..., 1] + 1) / 2 * (H - 1)).clamp(0, H - 1)
    return ix, iy


def bilinear(feats, ix, iy, swap=False):
    """float64 bilinear sample of feats [B, C, H, W] at pixel coordinates (ix, iy) [B, Ho, Wo] with out-of-range corners dropped, the rule of
    grid_sample; swap=True exchanges the two top corner weights (a deliberately wrong sampler)."""
    B, C, H, W = feats.shape
    x0, y0 = torch.floor(ix), torch.floor(iy)
    fx, fy = ix - x0, iy - y0
    wts = [(1 - fx) * (1 - fy), fx * (1 - fy), (1 - fx) * fy, fx * fy]
    if swap:
        wts[0], wts[1] = wts[1], wts[0]
    out = torch.zeros(B, C, *ix.shape[1:], dtype=torch.float64)
    flat = feats.double().reshape(B, C, H * W)
    for (dy, dx), wt in zip(((0, 0), (0, 1), (1, 0), (1, 1)), wts):
        yy, xx = y0 + dy, x0 + dx
        ok = (yy >= 0) & (yy <= H - 1) & (xx >= 0) & (xx <= W - 1)
        idx = (yy.clamp(0, H - 1) * W + xx.clamp(0, W - 1)).long().reshape(B, 1, -1).expand(B, C, -1)
        v = torch.gather(flat, 2, idx).reshape(out.shape)
        out = out + torch.where(ok[:, None], wt[:, None] * v, torch.zeros_like(v))
    return out


def lg_ref(x, dconv, P2, elev):
    """float64 grid_sample(cat[disparity, x], flow, bilinear, border, align_corners=True) with flow and disparity in float32 as above.
    Returns (sampled [B, C + 1, H, W] in the kernel's channel order x..., disparity; S = the same sample of |feats|; M = max |feats| per
    (image, channel), [B, C + 1, 1, 1])."""
    B, C, H, W = x.shape
    flow = lg_flow(dconv, P2, H, W, elev)
    feats = torch.cat([lg_disparity(P2, H, W, elev), x.float()], 1).double()
    kw = dict(mode="bilinear", padding_mode="border", align_corners=True)
    out = F.grid_sample(feats, flow.double(), **kw)
    S = F.grid_sample(feats.abs(), flow.double(), **kw)
    M = feats.abs().amax(dim=(2, 3), keepdim=True)
    perm = list(range(1, C + 1)) + [0]
    return out[:, perm], S[:, perm], M[:, perm]


def lg_coord_slack(H, W):
    """Pixels the device's sampling position may sit from the reference's.  Both compute the normalised grid in float32 in the same op order,
    but the device may contract -1 + step * i and the disparity term into fmas, its tanhf differs from torch's by a few ulps, and it
    unnormalises in float32 (3 roundings) where the reference does so in float64.  Each is a few ulps of a value below max(H, W);
    32 u max(H, W) covers them with margin and is still 5 orders below a pixel."""
    return 32 * U * max(H, W)


def lg_bound(S, M, H, W):
    """|device - reference| per element: 16 u S for the weights, the 4-term sum and the disparity's own float32 arithmetic, plus
    2 slack M: a position error of `slack` pixels in x and in y moves a bilinear sample by at most slack * M per axis."""
    return 16 * U * S + 2 * lg_coord_slack(H, W) * M


def trunc13(t):
    """t with its 13 low mantissa bits cleared (the part the tf32 MMA sees)"""
    return (t.contiguous().view(torch.int32) & -8192).view(torch.float32)


# ---------------------------------------------------------------------------------------------------------------------------------------
# fp16 (hi, lo) splitter and the tf32 lo splitter
# ---------------------------------------------------------------------------------------------------------------------------------------
FP16_OVERFLOW = 65520.0                          # smallest magnitude that rounds to inf in fp16 (round to nearest even)


def fp16_ties():
    """float32 values exactly halfway between two adjacent fp16 values, in the normal range at several exponents and in the subnormal range,
    with an even and an odd lower neighbour each (so both directions of round-to-even occur); negated copies included."""
    vals = []
    for e in (-14, -8, -1, 0, 3, 10, 15):
        ulp = 2.0 ** (e - 10)
        for m in (1024, 1025, 1500, 1501, 2046):          # m 2^(e-10) is an fp16 value; m = 2046 at e = 15: the tie below 65504
            vals.append((m + 0.5) * ulp)
    for k in (0, 1, 2, 3, 512, 1022, 1023):                # subnormal: k 2^-24, tie (k + 1/2) 2^-24 (k = 0: 2^-25 rounds to 0)
        vals.append((k + 0.5) * 2.0 ** -24)
    return vals + [-v for v in vals]


def fp16_specials():
    """in-range values the splitter must handle exactly: signed zeros, fp16 subnormals and the values below them, the top of the fp16 range
    (65504 <= |v| < 65520 rounds to +-65504 with no overflow), and values with bits far below the fp16 mantissa"""
    vals = [0.0, -0.0, 2.0 ** -24, -(2.0 ** -24), 3 * 2.0 ** -24, 2.0 ** -25 + 2.0 ** -30, 2.0 ** -26, 2.0 ** -14 - 2.0 ** -24,
            2.0 ** -14, 2.0 ** -30, -(2.0 ** -25 + 2.0 ** -27), 65504.0, -65504.0, 65519.0, -65519.0, 65519.99609375, 65510.5, 1.0 + 2.0 ** -23, 1.0 - 2.0 ** -24,
            3.140625 + 2.0 ** -21, -(2.71875 + 2.0 ** -19), 1234.5 + 2.0 ** -12, 2.0 ** -14 + 2.0 ** -23]
    return vals


def fp16_overflows():
    """values at or beyond the fp16 range: hi = +-inf, and the device raises the range flag"""
    return [65520.0, -65520.0, 65536.0, 70000.0, -1e6, 3e38]


def split_h16_ref(t):
    hi = t.half()
    return hi, (t - hi.float()).half()


def to_channels(vals, C):
    """a 1-D list of values -> float32 [npix, C] (zero padded), npix = ceil(len / C)"""
    t = torch.tensor(vals, dtype=torch.float64).float()
    n = -(-t.numel() // C)
    out = torch.zeros(n * C)
    out[:t.numel()] = t
    return out.reshape(n, C)
