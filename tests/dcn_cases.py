"""A float64 restatement of (modulated) deformable convolution, forward and backward, written from the reference's kernel rules, and
constructed offset families that put the sampling positions where the device code branches.

The rules (deform_conv_cuda_kernel.cu of the reference; csrc/dcn.cu, csrc/dcn_fused.cu and csrc/dcn_backward.cu follow them):
  * the sampling position of tap (kh, kw) of output pixel (ho, wo) is h = (float)(ho*s - pad + kh*dil) + dh, computed in FLOAT32 (the
    device and the reference add the offset to the integer base in float32); everything after it is float64 here;
  * a tap is valid iff h > -1 && w > -1 && h < H && w < W; the low corner is floor(h), and each of the four corners is zero outside the image;
  * at an integer h the bilinear weight of the row below is 0, so the derivative is one-sided (toward h + 1) and zero past the last row;
  * the coordinate and mask gradients of an invalid tap are zero.  That includes h == -1 exactly, where torchvision keeps the tap and
    returns a non-zero d/dh: torchvision serves as a cross-check of the forward only (test_dcn_cases_cpu.py).

Layouts are the reference's: x [B, C, H, W]; offset [B, 2*K*dg, Ho, Wo] with channel g*2K + 2k = dh and + 1 = dw of tap k in deformable
group g; mask [B, K*dg, Ho, Wo] (values, already through the sigmoid); weight [Cout, C, KH, KW].  `cols` is [B, Ho, Wo, K*C] in the device's
tap-major column order k*C + c.  Every function is vectorised torch and runs on the device of its inputs.

Each result comes with `abs_*`: the same sum over |terms| (|weights| x |corner values| x |mask| ...), the scale the tolerances of the tests
are expressed in.

Families (`FAMILIES`, built by `family_offsets`): zero, integer, half, knife, far, mask_extreme, random.  `boundary_offsets` builds a field
whose every tap sits exactly on the validity boundary (-1 or H / W).
"""
import torch

FAMILIES = ("zero", "integer", "half", "knife", "far", "mask_extreme", "random")
KNIFE_EPS = 2.0 ** -10


def out_hw(H, W, KH, KW, stride, pad, dil):
    return (H + 2 * pad - (dil * (KH - 1) + 1)) // stride + 1, (W + 2 * pad - (dil * (KW - 1) + 1)) // stride + 1


def base_positions(Ho, Wo, KH, KW, stride, pad, dil):
    """Integer base positions of every tap: bh [K, Ho], bw [K, Wo] (int64)."""
    k = torch.arange(KH * KW)
    bh = torch.arange(Ho)[None, :] * stride - pad + (k // KW)[:, None] * dil
    bw = torch.arange(Wo)[None, :] * stride - pad + (k % KW)[:, None] * dil
    return bh, bw


def positions(offset, KH, KW, stride, pad, dil, dg, exact=False):
    """Sampling positions h, w [B, dg, K, Ho, Wo] (float64).  exact=False: base + offset rounded to float32, as the device computes it;
    exact=True: in float64 (the finite-difference check, which perturbs offsets below float32 resolution)."""
    B, _, Ho, Wo = offset.shape
    K = KH * KW
    off = offset.reshape(B, dg, K, 2, Ho, Wo)
    bh, bw = base_positions(Ho, Wo, KH, KW, stride, pad, dil)
    bh, bw = bh.to(offset.device)[None, None, :, :, None], bw.to(offset.device)[None, None, :, None, :]
    if exact:
        return bh.double() + off[:, :, :, 0].double(), bw.double() + off[:, :, :, 1].double()
    return (bh.float() + off[:, :, :, 0].float()).double(), (bw.float() + off[:, :, :, 1].float()).double()


def _sampling(x, h, w):
    """Per tap: validity, the four corners' (flat index, bilinear weight, inside) and the fractions."""
    H, W = x.shape[2], x.shape[3]
    valid = (h > -1) & (w > -1) & (h < H) & (w < W)
    hl, wl = torch.floor(h), torch.floor(w)
    lh, lw = h - hl, w - wl
    hh, hw = 1 - lh, 1 - lw
    corners = []
    for dy, dx, wt in ((0, 0, hh * hw), (0, 1, hh * lw), (1, 0, lh * hw), (1, 1, lh * lw)):
        y, xx = hl + dy, wl + dx
        inside = valid & (y >= 0) & (y <= H - 1) & (xx >= 0) & (xx <= W - 1)
        idx = (y.clamp(0, H - 1) * W + xx.clamp(0, W - 1)).long()
        corners.append((idx, torch.where(inside, wt, torch.zeros_like(wt)), inside))
    return valid, corners, (lh, lw, hh, hw)


def _gather(x, dg, idx, inside):
    """x [B, C, H, W] at the corner `idx` [B, dg, K, Ho, Wo] -> [B, dg, cpg, K, Ho, Wo]; zero (not 0 * x) where the corner is outside."""
    B, C, H, W = x.shape
    cpg = C // dg
    sh = idx.shape
    flat = idx.reshape(B, dg, 1, -1).expand(B, dg, cpg, idx[0, 0].numel())
    v = torch.gather(x.reshape(B, dg, cpg, H * W), 3, flat).reshape(B, dg, cpg, *sh[2:])
    return torch.where(inside[:, :, None], v, torch.zeros_like(v))


def _mask(mask, h, dg):
    if mask is None:
        return torch.ones_like(h)
    B, _, Ho, Wo = mask.shape
    return mask.reshape(B, dg, -1, Ho, Wo).double()


def forward(x, offset, mask, weight, bias, stride, pad, dil, dg, exact=False):
    """Deformable conv (v2 with `mask`, v1 without).  Returns dict(out [B, Cout, Ho, Wo], abs_out, cols [B, Ho, Wo, K*C], abs_cols, h, w, valid)."""
    x = x.double()
    B, C, H, W = x.shape
    Cout, _, KH, KW = weight.shape
    K, cpg = KH * KW, C // dg
    h, w = positions(offset, KH, KW, stride, pad, dil, dg, exact)
    valid, corners, _ = _sampling(x, h, w)
    m = _mask(mask, h, dg)[:, :, None]                                  # [B, dg, 1, K, Ho, Wo]
    bil = 0.0
    abil = 0.0
    for idx, wt, inside in corners:
        v = _gather(x, dg, idx, inside)
        bil = bil + wt[:, :, None] * v
        abil = abil + wt[:, :, None].abs() * v.abs()
    cols, acols = m * bil, m.abs() * abil                               # [B, dg, cpg, K, Ho, Wo]
    wr = weight.double().reshape(Cout, dg, cpg, K)
    out = torch.einsum("bgckhw,ogck->bohw", cols, wr)
    aout = torch.einsum("bgckhw,ogck->bohw", acols, wr.abs())
    if bias is not None:
        out = out + bias.double()[None, :, None, None]
        aout = aout + bias.double().abs()[None, :, None, None]
    Ho, Wo = h.shape[3], h.shape[4]
    to_nhwc = lambda t: t.permute(0, 4, 5, 3, 1, 2).reshape(B, Ho, Wo, K * C)
    return dict(out=out, abs_out=aout, cols=to_nhwc(cols), abs_cols=to_nhwc(acols), h=h, w=w, valid=valid)


def backward(x, offset, mask, weight, grad_out, stride, pad, dil, dg, exact=False):
    """Gradients of sum(grad_out * forward(...)): dict(grad_input, grad_offset, grad_mask (None for v1), grad_weight, grad_bias), each with
    `abs_<name>` (the sum over |terms|), `count_input` (contributions per input element) and `edge` (bool, like grad_offset: the entries whose
    coordinate is exactly -1, where the reference's coordinate gradient is zero and torchvision's is not)."""
    x = x.double()
    g = grad_out.double()
    B, C, H, W = x.shape
    Cout, _, KH, KW = weight.shape
    K, cpg = KH * KW, C // dg
    h, w = positions(offset, KH, KW, stride, pad, dil, dg, exact)
    Ho, Wo = h.shape[3], h.shape[4]
    valid, corners, (lh, lw, hh, hw) = _sampling(x, h, w)
    m = _mask(mask, h, dg)
    wr = weight.double().reshape(Cout, dg, cpg, K)
    cg = torch.einsum("bohw,ogck->bgckhw", g, wr)                          # column gradient
    acg = torch.einsum("bohw,ogck->bgckhw", g.abs(), wr.abs())
    gx = torch.zeros(B, dg, cpg, H * W, dtype=torch.float64, device=x.device)
    agx = torch.zeros_like(gx)
    cnt = torch.zeros(B, dg, 1, H * W, dtype=torch.float64, device=x.device)
    zero = torch.zeros_like(h)
    coef_h = (-hw, -lw, hw, lw)                                            # d(bilinear)/dh per corner
    coef_w = (-hh, hh, -lh, lh)
    dh = dw = bil = adh = adw = abil = 0.0
    for n, (idx, wt, inside) in enumerate(corners):
        flat = idx.reshape(B, dg, 1, -1).expand(B, dg, cpg, idx[0, 0].numel())
        gx.scatter_add_(3, flat, (wt * m)[:, :, None].expand_as(cg).reshape(B, dg, cpg, -1) * cg.reshape(B, dg, cpg, -1))
        agx.scatter_add_(3, flat, (wt * m).abs()[:, :, None].expand_as(cg).reshape(B, dg, cpg, -1) * acg.reshape(B, dg, cpg, -1))
        cnt.scatter_add_(3, idx.reshape(B, dg, 1, -1), inside.double().reshape(B, dg, 1, -1))
        v = _gather(x, dg, idx, inside)
        ch = torch.where(valid, coef_h[n], zero)[:, :, None]
        cw = torch.where(valid, coef_w[n], zero)[:, :, None]
        dh, adh = dh + ch * v, adh + ch.abs() * v.abs()
        dw, adw = dw + cw * v, adw + cw.abs() * v.abs()
        bil, abil = bil + wt[:, :, None] * v, abil + wt[:, :, None].abs() * v.abs()
    goff = torch.stack([(cg * dh).sum(2) * m, (cg * dw).sum(2) * m], 3)            # [B, dg, K, 2, Ho, Wo]
    agoff = torch.stack([(acg * adh).sum(2) * m.abs(), (acg * adw).sum(2) * m.abs()], 3)
    cols, acols = m[:, :, None] * bil, m.abs()[:, :, None] * abil
    gw = torch.einsum("bohw,bgckhw->ogck", g, cols).reshape(Cout, C, KH, KW)
    agw = torch.einsum("bohw,bgckhw->ogck", g.abs(), acols).reshape(Cout, C, KH, KW)
    edge = torch.stack([(h == -1) & (w > -1) & (w < W), (w == -1) & (h > -1) & (h < H)], 3)
    r = dict(grad_input=gx.reshape(B, C, H, W), abs_grad_input=agx.reshape(B, C, H, W),
             count_input=cnt.expand(B, dg, cpg, H * W).reshape(B, C, H, W),
             grad_offset=goff.reshape(B, 2 * K * dg, Ho, Wo), abs_grad_offset=agoff.reshape(B, 2 * K * dg, Ho, Wo),
             edge=edge.reshape(B, 2 * K * dg, Ho, Wo),
             grad_weight=gw, abs_grad_weight=agw, grad_bias=g.sum((0, 2, 3)), abs_grad_bias=g.abs().sum((0, 2, 3)),
             grad_mask=None, abs_grad_mask=None)
    if mask is not None:
        r["grad_mask"] = ((cg * bil).sum(2) * valid).reshape(B, K * dg, Ho, Wo)
        r["abs_grad_mask"] = (acg * abil).sum(2).reshape(B, K * dg, Ho, Wo)
    return r


# ---- offset families --------------------------------------------------------------------------------------------------------------------
def _f32_exact(base, target):
    """dh with float32(base + dh) == target exactly (base: integer tensor, target: float64 tensor of float32 values)."""
    d = (target - base.double()).float()
    got = (base.float() + d).double()
    assert torch.equal(got, target), "knife target missed in float32"
    return d


def family_offsets(family, B, H, W, KH, KW, stride, pad, dil, dg, seed=0):
    """(offset [B, 2*K*dg, Ho, Wo], mask logits [B, K*dg, Ho, Wo]), both float32 on the CPU, for one family:
      zero          offsets 0, logits 0 (where training starts: the reference zero-inits conv_offset);
      integer       per-entry offsets in {+-1, +-2, +-3}: corners on integers, on and one pixel past the staged kernel's 2-pixel halo;
      half          +-0.5, +-1.5: every bilinear weight exactly 0.25 or 0.5;
      knife         float32 positions exactly -1, -1 + 2^-10, H - 1, H - 2^-10 or H (likewise for w), asserted exact;
      far           +-40.375 and beyond the image on both sides: positions entirely outside;
      mask_extreme  random offsets, logits +-20 and +-90 (sigmoid exactly 0 or 1 in float32; expf(90) overflows);
      random        randn * 2 offsets, randn logits (the random inputs of the older tests)."""
    assert family in FAMILIES, family
    Ho, Wo = out_hw(H, W, KH, KW, stride, pad, dil)
    K = KH * KW
    g = torch.Generator().manual_seed(1000 * seed + FAMILIES.index(family))
    shp = (B, dg, K, 2, Ho, Wo)
    logit = torch.randn(B, K * dg, Ho, Wo, generator=g)
    pick = lambda vals, n: torch.tensor(vals, dtype=torch.float32)[torch.randint(len(vals), n, generator=g)]
    if family == "zero":
        off, logit = torch.zeros(shp), torch.zeros_like(logit)
    elif family == "integer":
        off = pick([-3.0, -2.0, -1.0, 1.0, 2.0, 3.0], shp)
    elif family == "half":
        off = pick([-1.5, -0.5, 0.5, 1.5], shp)
    elif family == "knife":
        bh, bw = base_positions(Ho, Wo, KH, KW, stride, pad, dil)
        th = torch.tensor([-1.0, -1.0 + KNIFE_EPS, H - 1.0, H - KNIFE_EPS, float(H)], dtype=torch.float64)
        tw = torch.tensor([-1.0, -1.0 + KNIFE_EPS, W - 1.0, W - KNIFE_EPS, float(W)], dtype=torch.float64)
        ih = torch.randint(5, (B, dg, K, Ho, Wo), generator=g)
        iw = torch.randint(5, (B, dg, K, Ho, Wo), generator=g)
        # a third of the taps keep one coordinate at its regular position, so a knife coordinate meets a valid other one
        keep = torch.randint(3, (B, dg, K, Ho, Wo), generator=g)
        bhx, bwx = bh[None, None, :, :, None].expand(B, dg, K, Ho, Wo), bw[None, None, :, None, :].expand(B, dg, K, Ho, Wo)
        eh = torch.where(keep == 1, bhx.double().clamp(0, H - 1), th[ih])
        ew = torch.where(keep == 2, bwx.double().clamp(0, W - 1), tw[iw])
        off = torch.stack([_f32_exact(bhx, eh), _f32_exact(bwx, ew)], 3)
    elif family == "far":
        off = pick([-40.375, 40.375, -(H + W + 5.5), H + W + 5.5], shp)
        near = torch.rand(shp, generator=g) < 0.25               # some entries stay near, so one coordinate can be valid
        off = torch.where(near, torch.round(torch.randn(shp, generator=g) * 8) / 8, off)
    elif family == "mask_extreme":
        off = torch.randn(shp, generator=g) * 2.0
        logit = pick([-90.0, -20.0, 20.0, 90.0], tuple(logit.shape))
    else:
        off = torch.randn(shp, generator=g) * 2.0
    return off.reshape(B, 2 * K * dg, Ho, Wo).contiguous(), logit.contiguous()


def boundary_offsets(B, H, W, KH, KW, stride, pad, dil, dg):
    """Offsets that put every tap exactly on the validity boundary, cycling through (h, w) = (-1, 0.5), (0.5, -1), (H, 0.5), (0.5, W): no tap is
    valid, so the output is the bias whatever the image holds.  A tap at exactly -1 taken as valid would read row 0 / column 0 with weight 0."""
    assert H >= 2 and W >= 2
    Ho, Wo = out_hw(H, W, KH, KW, stride, pad, dil)
    K = KH * KW
    bh, bw = base_positions(Ho, Wo, KH, KW, stride, pad, dil)
    bhx = bh[None, None, :, :, None].expand(B, dg, K, Ho, Wo)
    bwx = bw[None, None, :, None, :].expand(B, dg, K, Ho, Wo)
    sel = (torch.arange(B * dg * K * Ho * Wo) % 4).reshape(B, dg, K, Ho, Wo)
    th = torch.stack([torch.full((), -1.0), torch.full((), 0.5), torch.full((), float(H)), torch.full((), 0.5)]).double()[sel]
    tw = torch.stack([torch.full((), 0.5), torch.full((), -1.0), torch.full((), 0.5), torch.full((), float(W))]).double()[sel]
    off = torch.stack([_f32_exact(bhx, th), _f32_exact(bwx, tw)], 3)
    return off.reshape(B, 2 * K * dg, Ho, Wo).contiguous()


def effective_offsets(offset, KH, KW, stride, pad, dil, dg):
    """float64 offsets whose float64 positions equal the float32 positions of `offset`: hands the device's positions to a float64 oracle."""
    B, _, Ho, Wo = offset.shape
    K = KH * KW
    h, w = positions(offset, KH, KW, stride, pad, dil, dg)
    bh, bw = base_positions(Ho, Wo, KH, KW, stride, pad, dil)
    bh, bw = bh.to(offset.device)[None, None, :, :, None].double(), bw.to(offset.device)[None, None, :, None, :].double()
    return torch.stack([h - bh, w - bw], 3).reshape(B, 2 * K * dg, Ho, Wo)


def sigmoid_f32(logit):
    """The device's mask: 1 / (1 + expf(-m)) in float32 (exactly 0 / 1 at the extreme logits)."""
    l = logit.float()
    return (1.0 / (1.0 + torch.exp(-l))).float()
