"""Float64 restatements of Stereo3D's two cost volumes, constructed operands with exact answers, the error bounds of the device paths, and
perturbed restatements that model the index errors the kernels could make.

The rules (R/lib/PSM_cost_volume.py; oracle/torch_port.py psm_cosine / concat_volume follow them):
  * PSMCosine: cost[b, h, w, d] = (1/C) sum_c L[b, h, w, c] * R[b, h, w - d, c] for w >= d, exactly 0 for w < d (planes d >= W are all 0);
  * concat volume: plane d holds cat[L[w], R[w - d]] for w >= d and 0 elsewhere, [B, 2F, D, H, W]; then Conv3d(2F -> F, 3, pad 1) + ReLU and
    Conv3d(F -> F, 3, pad 1) + ReLU (batch norm folded into the weights).  The device writes the result NHWC with channel f * D + d.
Operands and results here are in the device's NHWC layout: L, R [B, H, W, C] and the PSMCosine volume [B, H, W, D].  Every function is
vectorised torch and runs on the device of its inputs.

Constructed operands (`tag_features`, `tag_conv_operands`).  Integers with |v| <= 8: the fp16 hi plane of the tensor-core path holds each
value exactly and the lo plane is exactly 0 (asserted by `assert_exact_split`); every partial sum is an integer below 2^24, so every fp32
sum is exact in any order.  Each pixel's vector is drawn independently, so L[q] . R[q - d] depends on the source pixel (image, row, column):
a read of the wrong R pixel, disparity, tile or image changes the answer, which test_cost_volume_cases_cpu.py proves for every perturbation
below.  With C a power of two the scale 1/C is exact too; `device_scale` states the one rounding left for other C (most kernels multiply by
the fp32 reciprocal, the generic one and the NCHW mirror divide).  The device result of a tag case must therefore equal the restatement bit for bit, on every path.

Error bounds for random fp32 operands, per output element, with u = 2^-24 and S = sum_c |L| |R| / C (`psm_cosine64` returns S):
  * tensor-core path (`tc_bound`).  The operands are split as x = hi + lo + e with hi = rn16(x), lo = rn16(x - hi): |x - hi| <= 2^-11 |x|,
    so |lo| <= 2^-11 |x| (1 + 2^-11) and |e| <= 2^-22 |x| (lo normal) or 2^-25 absolute (lo in the fp16 subnormal range).  The kernel
    computes hi*hi + hi*lo + lo*hi and drops lo*lo (<= 2^-22 |L||R|); with e_L R and L e_R that is 3 * 2^-22 = 12 u per term, 13 u with the
    second-order factors, plus 2^-25 (|L| + |R|) per term from subnormal lo planes, which `tc_bound` takes as 2^-25 (max|L| + max|R|) per
    element after the 1/C average.  Products of fp16 values are exact in fp32.  A term then passes through at most 16 additions inside one
    wgmma (K = 16) and one accumulator update per later wgmma: 3 MMAs x 4 k-steps x C/64 k-blocks = 3C/16.  The tensor core may truncate
    rather than round, so each addition counts 2 u: (2 (3C/16 + 16) + 13 + 2) u S, the last 2 u for the fp32 reciprocal and the product with
    it.  At C = 64 that is 71 u ~ 2^-17.8 relative to S; a dropped lo plane (2^-11 per term) is far outside it.
  * SIMT paths (`simt_bound`): IEEE fp32 fma chains.  The deepest is the generic kernel's and the NCHW mirror's, C fmas per output (v2, v3
    and v4 use C/8 fmas and three shuffle adds); plus the scale: gamma(C + 1) S with gamma(n) = n u / (1 - n u), about C 2^-24 relative.
  * concat volume + Conv3d pair (`concat_conv3d64` returns the bound): the volume is gathered exactly; Conv3d #1 is 27 taps x 16 channels
    = 432 fmas and the bias add, gamma(433) A1 with A1 = conv(|vol|, |w1|) + |b1|; the ReLU does not increase an error; Conv3d #2 sees that
    error through |w2| and adds its own 216 fmas and bias, gamma(217) A2 with A2 = conv(|mid|, |w2|) + |b2|:
    bound = (1 + gamma(217)) conv(gamma(433) A1, |w2|) + gamma(217) A2.
These are worst-case rounding counts, not fits to measured errors.

Perturbations (the keyword arguments of the restatements, `swap_tiles`, `swap_images`): R read one pixel left or right (`r_shift`), the
value of disparity d + 1 stored at d (`d_shift`), the mask w >= d replaced by w > d (`strict`), two 128-pixel tensor-core tiles swapped,
two images of the batch swapped.
"""
import math

import torch
import torch.nn.functional as F

U = 2.0 ** -24
TC_TILE = 128                  # pixels per tile of the tensor-core kernel (flat across rows and images)
TAG_MAX = 8


def gamma(n):
    return n * U / (1.0 - n * U)


def assert_exact_split(x):
    """The fp16 (hi, lo) split of the tensor-core path holds x exactly in hi and leaves lo exactly 0."""
    hi = x.half()
    lo = (x.float() - hi.float()).half()
    assert torch.equal(hi.float(), x.float()) and not bool(lo.any()), "tag operand not exact in fp16"


def tag_features(B, H, W, C, seed):
    """Integer L, R [B, H, W, C] in [1, TAG_MAX] (float32, CPU).  Positive, so every product sum is at least C: the w == d column never
    holds a 0 that a w > d mask would also produce."""
    g = torch.Generator().manual_seed(seed)
    L = torch.randint(1, TAG_MAX + 1, (B, H, W, C), generator=g).float()
    R = torch.randint(1, TAG_MAX + 1, (B, H, W, C), generator=g).float()
    assert C * TAG_MAX * TAG_MAX < 2 ** 24, "partial sums would leave the exact fp32 integers"
    assert_exact_split(L), assert_exact_split(R)
    return L, R


def random_features(B, H, W, C, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, H, W, C, generator=g), torch.randn(B, H, W, C, generator=g)


def shift_w(x, s):
    """x'[..., w, :] = x[..., w + s, :] along the width of an NHWC tensor, 0 outside."""
    out = torch.zeros_like(x)
    W = x.shape[2]
    if s >= 0:
        out[:, :, :W - s] = x[:, :, s:]
    else:
        out[:, :, -s:] = x[:, :, :W + s]
    return out


def _columns(W, d, d_shift, strict):
    """Columns [lo, hi) of disparity plane d that hold a value, and the disparity `src` its R pixel is read at."""
    src = d + d_shift
    return max(d + 1 if strict else d, src, 0), min(W, W + src), src


def psm_cosine64(L, R, D, r_shift=0, d_shift=0, strict=False):
    """PSMCosine in float64: (cost [B, H, W, D], S [B, H, W, D] = sum_c |L| |R| / C).  The keyword arguments perturb it (module docstring)."""
    L, R = L.double(), R.double()
    B, H, W, C = L.shape
    if r_shift:
        R = shift_w(R, r_shift)
    out = L.new_zeros(B, H, W, D)
    S = L.new_zeros(B, H, W, D)
    for d in range(D):
        lo, hi, src = _columns(W, d, d_shift, strict)
        if lo >= hi:
            continue
        l, r = L[:, :, lo:hi], R[:, :, lo - src:hi - src]
        out[:, :, lo:hi, d] = (l * r).sum(-1) / C
        S[:, :, lo:hi, d] = (l.abs() * r.abs()).sum(-1) / C
    return out, S


def device_scale(cost, C, divide=False):
    """A tag case's exact float64 cost as the kernels produce it in float32 from the exact integer sum: times the fp32 reciprocal of C
    (tensor-core, v2, v3, v4) or divided by C (`divide`: the generic kernel and the NCHW mirror), rounded once.  Both equal cost itself when
    C is a power of two.  The divided form is the float64 quotient rounded to fp32: a quotient n / C of an integer n that is not an fp32
    value lies about 2^-24 / C (relative) away from every fp32 rounding midpoint, far beyond float64's 2^-53, so rounding twice cannot
    differ from the fp32 division's one correct rounding.  (torch's division of a float32 tensor by a scalar multiplies by the reciprocal
    on the GPU, so it cannot state the kernels' division.)"""
    if divide:
        return cost.float()
    inv = torch.tensor(1.0 / C, dtype=torch.float32, device=cost.device)
    return (cost * C).float() * inv


def tc_bound(C, S, L, R):
    n_acc = 3 * C // 16 + 16
    return (2 * n_acc + 13 + 2) * U * S + 2.0 ** -25 * (float(L.abs().max()) + float(R.abs().max()))


def simt_bound(C, S):
    return gamma(C + 1) * S


def swap_tiles(cost, t0, t1, tile=TC_TILE):
    """cost [B, H, W, D] with the flat pixel ranges of tiles t0 and t1 exchanged."""
    D = cost.shape[-1]
    flat = cost.reshape(-1, D).clone()
    a, b = slice(t0 * tile, (t0 + 1) * tile), slice(t1 * tile, (t1 + 1) * tile)
    assert flat[b].shape[0] == tile, "both tiles must be whole"
    flat[a], flat[b] = cost.reshape(-1, D)[b], cost.reshape(-1, D)[a]
    return flat.reshape(cost.shape)


def swap_images(x, b0, b1):
    y = x.clone()
    y[b0], y[b1] = x[b1], x[b0]
    return y


# ---- concat volume + Conv3d pair ----------------------------------------------------------------------------------------------------------
def concat_volume64(lf, rf, D, r_shift=0, d_shift=0, strict=False):
    """lf, rf [B, H, W, F] -> the concat volume [B, 2F, D, H, W] in float64."""
    lf, rf = lf.double(), rf.double()
    if r_shift:
        rf = shift_w(rf, r_shift)
    B, H, W, Fc = lf.shape
    L, R = lf.permute(0, 3, 1, 2), rf.permute(0, 3, 1, 2)
    vol = lf.new_zeros(B, 2 * Fc, D, H, W)
    for d in range(D):
        lo, hi, src = _columns(W, d, d_shift, strict)
        if lo >= hi:
            continue
        vol[:, :Fc, d, :, lo:hi] = L[..., lo:hi]
        vol[:, Fc:, d, :, lo:hi] = R[..., lo - src:hi - src]
    return vol


def conv3d64(x, w, b):
    """3x3x3 convolution, padding 1, as a sum over the 27 taps in float64 (x [B, Ci, D, H, W], w [Co, Ci, 3, 3, 3])."""
    B, _, D, H, W = x.shape
    xp = F.pad(x.double(), (1, 1, 1, 1, 1, 1))
    w = w.double()
    out = b.double().reshape(1, -1, 1, 1, 1).expand(B, w.shape[0], D, H, W).clone()
    for kd in range(3):
        for kh in range(3):
            for kw in range(3):
                out += torch.einsum("bcdhw,oc->bodhw", xp[:, :, kd:kd + D, kh:kh + H, kw:kw + W], w[:, :, kd, kh, kw])
    return out


def to_device_layout(y):
    """[B, F, D, H, W] -> [B, H, W, F * D] with channel f * D + d."""
    B, Fc, D, H, W = y.shape
    return y.permute(0, 3, 4, 1, 2).reshape(B, H, W, Fc * D)


def concat_conv3d64(lf, rf, w1, b1, w2, b2, D, **perturb):
    """Concat volume + Conv3d + ReLU + Conv3d + ReLU in float64.  Returns dict(out [B, H, W, F * D], mid [B, F, D, H, W], bound, abs_max):
    `bound` the fp32 bound of the module docstring, `abs_max` the largest sum over |terms| of either layer (exactness needs < 2^24)."""
    vol = concat_volume64(lf, rf, D, **perturb)
    mid = torch.relu(conv3d64(vol, w1, b1))
    out = torch.relu(conv3d64(mid, w2, b2))
    a1 = conv3d64(vol.abs(), w1.abs(), b1.abs())
    a2 = conv3d64(mid, w2.abs(), b2.abs())
    e1 = gamma(433) * a1
    bound = (1 + gamma(217)) * conv3d64(e1, w2.abs(), torch.zeros_like(b2)) + gamma(217) * a2
    return dict(out=to_device_layout(out), mid=mid, bound=to_device_layout(bound), abs_max=max(float(a1.max()), float(a2.max())))


def pack_conv3d(w):
    """[Co, Ci, 3, 3, 3] -> the device layout [27, Ci, Co] (Stereo3D.build_plan packs the folded weights the same way)."""
    return w.permute(2, 3, 4, 1, 0).reshape(27, w.shape[1], w.shape[0]).contiguous()


def tag_conv_operands(B, H, W, Fc, seed):
    """Integer features in [-4, 4], weights in [-2, 2], biases in [-8, 8] (float32, CPU): both layers' sums are integers below 2^24, so the
    device result, ReLUs included, is exact.  Features and weights of both signs, so both ReLUs clip."""
    g = torch.Generator().manual_seed(seed)
    ri = lambda a, *shape: torch.randint(-a, a + 1, shape, generator=g).float()  # noqa: E731
    return (ri(4, B, H, W, Fc), ri(4, B, H, W, Fc), ri(2, Fc, 2 * Fc, 3, 3, 3), ri(8, Fc), ri(2, Fc, Fc, 3, 3, 3), ri(8, Fc))


def random_conv_operands(B, H, W, Fc, seed):
    """Non-negative features (the down-sample's ReLU output) and weights of the scale of a folded Conv3d."""
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(B, H, W, Fc, generator=g), torch.rand(B, H, W, Fc, generator=g),
            torch.randn(Fc, 2 * Fc, 3, 3, 3, generator=g) / math.sqrt(54 * Fc), torch.randn(Fc, generator=g) * 0.1,
            torch.randn(Fc, Fc, 3, 3, 3, generator=g) / math.sqrt(27 * Fc), torch.randn(Fc, generator=g) * 0.1)


# ---- the cases ----------------------------------------------------------------------------------------------------------------------------
def _case(id, B, H, W, C, D, cs=None, co=0, out_cs=None, out_co=0):
    return dict(id=id, B=B, H=H, W=W, C=C, D=D, cs=cs or C, co=co, out_cs=out_cs or D + 8, out_co=out_co if out_cs else 4)


# Tensor-core PSMCosine (vd3d_psm_cosine_h16 via engine.psm_cosine_stereo): grid = min(ceil(B*H*W / 128), 132) persistent CTAs.
# Production (384 x 1280 pair, Stereo3D): scale 4 = 96 x 320, C = 64, D4 = 24 into G4[0:24] of 72 channels; scale 8 = 48 x 160, C = 128,
# D8 = 24 into G8[72:96] of 288 channels.
TC_CASES = [_case(f"c{C}_d{D}", 2, 3, 50, C, D) for C in (64, 128, 192, 256) for D in (4, 8, 12, 24, 28, 32)] + [
    _case("s4_b1", 1, 96, 320, 64, 24, out_cs=72, out_co=0),               # 240 tiles: 1-2 per CTA
    _case("s4_b2", 2, 96, 320, 64, 24, out_cs=72, out_co=0),               # 480 tiles: 3-4 per CTA
    _case("s8_b1", 1, 48, 160, 128, 24, out_cs=288, out_co=72),
    _case("s8_b2", 2, 48, 160, 128, 24, out_cs=288, out_co=72),
    _case("c256_ragged", 2, 40, 220, 256, 24),                              # 137.5 tiles: 4 k-blocks per tile, ring wraps inside a CTA
    _case("npix_ragged", 3, 5, 37, 128, 12),                                # 555 pixels: tiles straddle rows and images
    _case("w_lt_d", 2, 9, 20, 64, 32),                                      # W < D, W < 32
    _case("w1", 2, 70, 1, 64, 8),
    _case("h1", 2, 1, 200, 64, 24),
    _case("seams", 2, 2, 96, 128, 28),                                      # tile 0 holds a row seam, tile 1 the image seam
    _case("chan_offset", 2, 6, 50, 64, 24, cs=88, co=16),                   # features at channels [16, 80) of 88
]

# SIMT PSMCosine (vd3d_psm_cosine_nhwc via engine.psm_cosine); `path` is the kernel the launch rules pick with the default variant.
SIMT_CASES = [
    dict(_case("v4_c64", 2, 96, 300, 64, 24), path="v4"),                   # 960 64-pixel tiles on 264 CTAs: 3-4 per CTA, W % 64 = 44
    dict(_case("v4_c128", 2, 48, 300, 128, 24), path="v4"),                 # 480 tiles on 132 CTAs
    dict(_case("v3_c64_sliced", 2, 5, 150, 64, 24, cs=72, co=4), path="v3"),
    dict(_case("v3_c128_sliced", 2, 5, 150, 128, 24, cs=136, co=4), path="v3"),
    dict(_case("generic_d1", 2, 4, 70, 32, 1, out_cs=8, out_co=3), path="generic"),
    dict(_case("generic_d12", 2, 4, 70, 32, 12, out_cs=20, out_co=3), path="generic"),
    dict(_case("generic_d64", 2, 4, 70, 32, 64, out_cs=72, out_co=3), path="generic"),
    dict(_case("generic_c64_odd_out", 1, 3, 40, 64, 24, out_cs=29, out_co=1), path="generic"),   # fast shape, output pitch not a multiple of 4
]

# Dense inputs, run by tests/workers/psm_variant.py under VD3D_PSM_VARIANT = 2 or 3 (the variant is read once per process).
VARIANT_CASES = [_case("c64", 2, 5, 150, 64, 24), _case("c128", 2, 5, 150, 128, 24), _case("c64_w_lt_d", 1, 3, 20, 64, 24)]

NCHW_CASES = [
    _case("nchw_d13", 2, 5, 40, 48, 13),                                    # C = 48: the division by C rounds
    _case("nchw_d24_w_lt_d", 1, 3, 17, 64, 24),
]


def _cv(id, B, H, W, D, out_cs=None, out_co=0):
    return dict(id=id, B=B, H=H, W=W, F=8, D=D, out_cs=out_cs or 8 * D + 8, out_co=out_co if out_cs else 4)


# Concat volume + Conv3d pair (vd3d_concat_volume_conv3d).  Production: scale 16 of a 384 x 1280 pair is 24 x 80 (6 x 20 at the test size
# 96 x 320), D16 = 12, F = 8; the volume is written into G16[3*c8 : 3*c8 + 96] of 3*c16 = 1152 channels (c8 = 96, c16 = 384).
CONCAT_CASES = [
    _cv("d1", 2, 6, 20, 1),
    _cv("d12_prod_6x20", 2, 6, 20, 12, out_cs=1152, out_co=288),
    _cv("d12_prod_24x80", 1, 24, 80, 12, out_cs=1152, out_co=288),
    _cv("d30_gt_w", 1, 4, 20, 30),
    _cv("h1", 2, 1, 40, 12),
    _cv("w1", 2, 5, 1, 12),
    _cv("b3", 3, 6, 20, 12),
]


def case_seed(case, salt=0):
    return sum(ord(ch) for ch in case["id"]) * 7 + salt
