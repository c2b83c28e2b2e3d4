"""-m gpu: the deformable convolution's device code on the constructed offset families of tests/dcn_cases.py, against its float64 restatement.

Paths: the fused gather + wgmma kernels of csrc/dcn_fused.cu (staged and global-gather, every BN instance, several units per CTA), the unfused
DeformConvLayer path (vd3d_deform_im2col_h16 + 1x1 conv), the `ops` API forward (vd3d_deform_im2col_nhwc + 3xTF32 conv) with its column tensor,
and the `ops` API backward (column-gradient GEMM, vd3d_deform_col2im_nhwc, weight-gradient GEMM).

Tolerances.  Every bound is |device - restatement| <= (n * u) * S + floor, per output element, with u = 2^-24 and S the restatement's sum over
|terms| of that element (dcn_cases.py `abs_*`); the assertion is on the ratio |error| / bound <= 1, and the largest ratio is printed per family
and path.  n counts float32 roundings on the longest path to the element:
  * column value m * sum_n w_n v_n (the gather): 4 bilinear weights (1 rounding each, 2 when 1 - l rounds), a 4-term fma chain, the mask
    product and the mask's sigmoid (3): at most 10; COL_N = 16.
  * fp16-split GEMM (fused kernels and the unfused 1x1 conv): each operand as hi + lo fp16 carries 2^-22 relative (the lo plane's rounding)
    plus 2^-25 absolute (lo below the fp16 normal range); the dropped lo * lo product is 2^-22: 12 u per term, plus FLOOR16 = 2^-24 * sum|W|
    per output.  Accumulation in float32: 3 MMAs x (64 / 16) k-steps x 4 k-blocks between promotions = 48 adds, 16 inside an MMA, one per
    promotion (ceil(KB / 4), KB = ceil(K*C / 32) as an upper bound on the k-blocks), 4 in the epilogue (scale, bias, residual).
  * 3xTF32 GEMM (the `ops` forward): hi = truncation to tf32 and lo = tf32(x - hi) leave 2^-20 relative per operand, plus the dropped lo * lo:
    48 u per term; the same accumulation count.
  * backward: the column gradient is an fp32 GEMM over Cout (Cout roundings; TF32 is switched off for these tests).  grad_input: the product
    w * m * colgrad (3) and one atomic add per contribution (`count_input`).  grad_offset / grad_mask: the d-weight combination (6), the
    channel-quad sum (3), the mask (1) and one shared-memory atomic per quad (C / dg / 4).  grad_weight: the columns (COL_N) and an fp32 GEMM
    over B*Ho*Wo.  grad_bias: a sum over B*Ho*Wo.
These are worst-case rounding counts, not fits to measured errors.  At the knife-edge entries (position exactly -1) grad_offset is asserted to
be exactly 0.0, the reference's rule.
"""
import math

import numpy as np
import pytest
import torch

import dcn_cases as dc
from visualdet3d_b200 import engine as E
from visualdet3d_b200._lib import call
from visualdet3d_b200.ops import dcn

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
COL_N = 16
NUM_SMS = 132                  # H100 SXM: the fused kernels' grid is min(units, 132)
TILE_H, TILE_W = 8, 16         # the fused kernels' output tile (TC_TH x TC_TW)


@pytest.fixture(autouse=True)
def _fp32_matmul():
    saved = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = saved


def acc_n(KC):
    return 48 + 16 + math.ceil(math.ceil(KC / 32) / 4) + 4


def check(got, want, bound, what):
    """max |got - want| / bound <= 1; returns the ratio."""
    got, want, bound = got.double(), want.double(), bound.double()
    assert torch.isfinite(got).all(), (what, "non-finite output")
    ratio = float(((got - want).abs() / bound).max()) if got.numel() else 0.0
    print(f"  {what}: max |err| / bound = {ratio:.2e}")
    assert ratio <= 1.0, (what, ratio)
    return ratio


# ---- DeformConvLayer with a given om --------------------------------------------------------------------------------------------------
def run_with_om(layer, x, om, out, arena, name, res=None):
    """The calls DeformConvLayer.__call__ makes after its offset conv, fed with `om` instead of the offset conv's output (NHWC, channels
    [0, 2*K*dg) offsets, [2*K*dg, 3*K*dg) mask logits).  test_run_with_om_is_the_layer pins it to the layer bit for bit."""
    B, K = x.B, layer.KH * layer.KW
    Ho, Wo = layer.out_hw(x.H, x.W)
    m = layer.main
    if layer.fused_ok():
        oh, ol = out.h16_ptrs
        out.f32 = True
        call("vd3d_deform_conv_fused", x.ptr, B, x.H, x.W, x.C, x.cs, x.co, om.ptr, om.cs, 0, 2 * K * layer.dg, 1, 1,
             layer.KH, layer.KW, layer.stride, layer.pad, layer.dil, layer.k_order, m.w_hi.data_ptr(), m.w_lo.data_ptr(), m.out_scale, m.b.data_ptr(),
             res.ptr if res is not None else None, res.cs if res is not None else 0, res.co if res is not None else 0,
             out.ptr, oh, ol, m.Cout, out.cs, out.co, 1 if m.relu else 0, E._stream())
        return out
    cols = arena.act("dcn.cols", (B, Ho, Wo, K * layer.C), x.t.device, lo=True)
    ch, cl = cols.h16_ptrs
    call("vd3d_deform_im2col_h16", x.ptr, B, x.H, x.W, x.C, x.cs, x.co, om.ptr, om.cs, 0, om.ptr, om.cs, 2 * K * layer.dg, 1,
         layer.KH, layer.KW, layer.stride, layer.pad, layer.dil, layer.dg, layer.k_order, cols.ptr if E.CHECK_LO else None, ch, cl, cols.cs,
         E._stream())
    return m(cols, out, res=res)


def make_layer(C, Co, k, s, p, d, dg, relu, seed, off_bias=None):
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(Co, C, k, k, generator=g) / np.sqrt(C * k * k)
    b = torch.randn(Co, generator=g)
    n = 3 * k * k * dg
    ob = torch.zeros(n) if off_bias is None else off_bias
    layer = E.DeformConvLayer(w, b, torch.zeros(n, C, k, k), ob, None, stride=s, pad=p, dil=d, deform_groups=dg, relu=relu, device="cuda")
    return layer, w, b


def planes(*shape, fill=0.0):
    return torch.full((2, *shape), fill, device="cuda", dtype=torch.float16)


def x_act(x):
    B, C, H, W = x.shape
    return E.split_lo(E.Act(x.permute(0, 2, 3, 1).contiguous().cuda(), 0, None, planes(B, H, W, C)))


def om_act(layer, off, logit):
    B, _, Ho, Wo = off.shape
    t = torch.zeros(B, Ho, Wo, layer.n_off_pad, device="cuda")
    n = off.shape[1]
    t[..., :n] = off.permute(0, 2, 3, 1).cuda()
    t[..., n:n + logit.shape[1]] = logit.permute(0, 2, 3, 1).cuda()
    return E.Act(t)


def layer_bound(r, w, res, KC):
    S = r["abs_out"] + (res.abs() if res is not None else 0.0)
    floor = 2.0 ** -24 * w.double().abs().sum((1, 2, 3)).cuda()[None, :, None, None]
    return (COL_N + 12 + acc_n(KC)) * U * S + floor


def layer_case(B, C, H, W, Co, k, s, p, d, dg, family, relu, seed, monkeypatch, variants, x=None, off=None, res_on=True):
    """Runs one layer on every (fused, staged) variant with the family's om; asserts bit-identity across variants, untouched neighbour
    channels, and the first variant against the restatement.  Returns (outputs, restatement, bound)."""
    layer, w, b = make_layer(C, Co, k, s, p, d, dg, relu, seed)
    Ho, Wo = layer.out_hw(H, W)
    g = torch.Generator().manual_seed(seed + 1)
    if x is None:
        x = torch.randn(B, C, H, W, generator=g)
    fam_off, logit = dc.family_offsets(family, B, H, W, k, k, s, p, d, dg, seed) if family else (None, torch.zeros(B, k * k * dg, Ho, Wo))
    off = fam_off if off is None else off
    xa, om = x_act(x), om_act(layer, off, logit)
    res = E.Act(torch.randn(B, Ho, Wo, Co, generator=g).cuda()) if res_on else None
    outs = []
    for fused, staged in variants:
        monkeypatch.setenv("VD3D_DCN_FUSED", fused)
        monkeypatch.setenv("VD3D_DCN_STAGED", staged)
        assert layer.fused_ok() == (fused == "1")
        out = E.Act(torch.full((B, Ho, Wo, Co + 8), 7.0, device="cuda"), 4, Co, planes(B, Ho, Wo, Co + 8, fill=7.0))
        run_with_om(layer, xa, om, out, E.Arena(), "t", res=res)
        torch.cuda.synchronize()
        outs.append((out.t.clone(), out.lo.clone()))
    for o in outs[1:]:
        assert torch.equal(outs[0][0], o[0]) and torch.equal(outs[0][1], o[1]), "variants differ"
    t, pl = outs[0]
    assert bool((t[..., :4] == 7.0).all()) and bool((t[..., 4 + Co:] == 7.0).all()), "neighbour channels written"
    assert bool((pl[..., :4] == 7.0).all()) and bool((pl[..., 4 + Co:] == 7.0).all()), "neighbour channels of the fp16 planes written"
    mask = torch.sigmoid(logit.double()).cuda()
    r = dc.forward(x.double().cuda(), off.cuda(), mask, w.cuda(), b.cuda(), s, p, d, dg)
    want = r["out"] + (res.t.permute(0, 3, 1, 2).double() if res_on else 0.0)
    if relu:
        want = want.clamp_min(0.0)
    got = t[..., 4:4 + Co].permute(0, 3, 1, 2)
    return got, want, layer_bound(r, w, res.t.permute(0, 3, 1, 2).double() if res_on else None, k * k * C), layer


def units(B, Ho, Wo, Co):
    cp = (Co + 15) // 16 * 16
    return B * math.ceil(Ho / TILE_H) * math.ceil(Wo / TILE_W) * math.ceil(cp / min(cp, 64))


# B, C, H, W, Cout, stride, dil: staged kernel (3x3, stride 1, pad 1)
STAGED = [(4, 64, 64, 160, 64, 1, 1), (1, 128, 21, 30, 128, 1, 1), (2, 256, 13, 21, 36, 1, 1), (1, 64, 3, 5, 16, 1, 1),
          (2, 64, 19, 27, 24, 1, 1), (1, 64, 11, 37, 48, 1, 1), (1, 128, 9, 18, 72, 1, 1)]
# global-gather kernel: stride 2 / dilation 2 (pad = dilation), and the staged shapes' layer with VD3D_DCN_STAGED=0
GLOBAL = [(2, 64, 33, 47, 72, 2, 1), (1, 192, 17, 30, 36, 1, 2), (1, 64, 3, 5, 16, 2, 1), (4, 64, 64, 160, 64, 1, 2), (1, 192, 10, 13, 24, 2, 1)]


@pytest.mark.parametrize("family", dc.FAMILIES)
@pytest.mark.parametrize("shape", STAGED + GLOBAL)
def test_fused_kernels_on_families(shape, family, monkeypatch):
    B, C, H, W, Co, s, d = shape
    staged = shape in STAGED
    variants = [("1", "1"), ("0", "1")] + ([("1", "0")] if (staged and C == 64) else [])
    if not staged:
        variants = [("1", "0"), ("0", "0")]
    idx = (STAGED + GLOBAL).index(shape)
    got, want, bound, layer = layer_case(B, C, H, W, Co, 3, s, d, d, 1, family, relu=idx % 2 == 0, seed=idx, monkeypatch=monkeypatch,
                                         variants=variants, res_on=idx % 3 != 2)
    assert layer.k_order == (1 if staged else 0)
    Ho, Wo = layer.out_hw(H, W)
    n_units = units(B, Ho, Wo, Co)
    if shape in ((4, 64, 64, 160, 64, 1, 1), (4, 64, 64, 160, 64, 1, 2)):
        assert n_units >= 2 * NUM_SMS                                   # every CTA runs at least two units
    if Co == 128:
        assert n_units == 2 * units(B, Ho, Wo, 64)                      # two n-tiles
    check(got, want, bound, f"{'staged' if staged else 'global'} {shape} {family} ({n_units} units)")


def test_run_with_om_is_the_layer(monkeypatch):
    """run_with_om against DeformConvLayer itself, bit for bit: zero offset-conv weights and constant per-tap offsets / logits as its bias, so
    the layer's own offset conv writes the om (the one read back from the arena feeds run_with_om)."""
    for (B, C, H, W, Co, k, s, p, d, dg, fused, staged) in ((2, 64, 13, 21, 48, 3, 1, 1, 1, 1, "1", "1"), (1, 64, 17, 19, 36, 3, 2, 1, 1, 1, "1", "0"),
                                                            (1, 32, 9, 14, 24, 5, 1, 2, 1, 2, "0", "1")):
        K = k * k
        g = torch.Generator().manual_seed(C + k)
        ob = torch.cat([torch.tensor([-1.5, 2.0, 0.25, -3.0, 0.0, 1.0] * (K * dg))[:2 * K * dg], torch.randn(K * dg, generator=g)])
        layer, w, b = make_layer(C, Co, k, s, p, d, dg, True, 5, off_bias=ob)
        monkeypatch.setenv("VD3D_DCN_FUSED", fused)
        monkeypatch.setenv("VD3D_DCN_STAGED", staged)
        x = torch.randn(B, C, H, W, generator=g)
        xa = x_act(x)
        Ho, Wo = layer.out_hw(H, W)
        res = E.Act(torch.randn(B, Ho, Wo, Co, generator=g).cuda())
        ar = E.Arena()
        o1 = E.Act(torch.zeros(B, Ho, Wo, Co, device="cuda"), 0, None, planes(B, Ho, Wo, Co))
        layer(xa, o1, ar, "t", res=res)
        om = E.Act(ar.get("t.om", (B, Ho, Wo, layer.n_off_pad), xa.t.device))
        o2 = E.Act(torch.zeros(B, Ho, Wo, Co, device="cuda"), 0, None, planes(B, Ho, Wo, Co))
        run_with_om(layer, xa, om, o2, E.Arena(), "t", res=res)
        torch.cuda.synchronize()
        assert torch.equal(o1.t, o2.t) and torch.equal(o1.lo, o2.lo)
        n = 3 * K * dg
        print(f"  offset conv returns its bias exactly: {torch.equal(om.t[..., :n].cpu(), ob.float().expand(B, Ho, Wo, n))}")


# ---- unfused gather: DeformConvLayer with deformable groups / other kernel sizes ---------------------------------------------------------
@pytest.mark.parametrize("family", dc.FAMILIES)
@pytest.mark.parametrize("shape", [(2, 32, 11, 13, 24, 1, 0), (1, 96, 9, 14, 40, 5, 2), (1, 32, 7, 10, 16, 5, 2)])
def test_unfused_layer_on_families(shape, family, monkeypatch):
    B, C, H, W, Co, k, p = shape
    got, want, bound, layer = layer_case(B, C, H, W, Co, k, 1, p, 1, 2, family, relu=False, seed=C + k, monkeypatch=monkeypatch,
                                         variants=[("0", "1")])
    monkeypatch.setenv("VD3D_DCN_FUSED", "1")
    assert not layer.fused_ok() and layer.k_order == 0                 # deformable groups: the fused kernels do not take the layer
    check(got, want, bound, f"unfused dg=2 {shape} {family}")


# ---- ops API forward and its column tensor ---------------------------------------------------------------------------------------------
OPS = [(2, 4, 9, 11, 6, 7, 1, 3, 1, 1), (1, 8, 12, 10, 5, 7, 1, 3, 1, 2), (1, 16, 13, 17, 4, 3, 2, 2, 2, 4), (2, 8, 3, 5, 3, 3, 1, 1, 1, 2)]


def ops_inputs(case, family, seed):
    B, C, H, W, Co, k, s, p, d, dg = case
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, C, H, W, generator=g)
    w = torch.randn(Co, C, k, k, generator=g) / np.sqrt(C * k * k)
    b = torch.randn(Co, generator=g)
    off, logit = dc.family_offsets(family, B, H, W, k, k, s, p, d, dg, seed)
    return x, w, b, off, dc.sigmoid_f32(logit)


@pytest.mark.parametrize("family", dc.FAMILIES)
@pytest.mark.parametrize("case", OPS)
def test_ops_forward_and_columns_on_families(case, family):
    B, C, H, W, Co, k, s, p, d, dg = case
    x, w, b, off, mask = ops_inputs(case, family, OPS.index(case))
    xc, wc, bc, oc, mc = x.cuda(), w.cuda(), b.cuda(), off.cuda(), mask.cuda()
    Ho, Wo = dc.out_hw(H, W, k, k, s, p, d)
    K = k * k
    e = xc.new_empty(0)
    for v2 in (True, False):
        r = dc.forward(xc.double(), oc, mc if v2 else None, wc, bc if v2 else None, s, p, d, dg)
        out = torch.empty(B, Co, Ho, Wo, device="cuda")
        if v2:
            dcn.modulated_deform_conv_forward(xc, wc, bc, e, oc, mc, out, e, k, k, s, s, p, p, d, d, 1, dg, True)
        else:
            assert dcn.deform_conv_forward(xc, wc, oc, out, e, e, k, k, s, s, p, p, d, d, 1, dg, B) == 1
        torch.cuda.synchronize()
        check(out, r["out"], (COL_N + 48 + acc_n(K * C)) * U * r["abs_out"] + 1e-30, f"ops {'v2' if v2 else 'v1'} {case} {family}")
        # the gather's column tensor on its own: a few roundings of the fma chain
        xn = x.permute(0, 2, 3, 1).contiguous().cuda()
        om = torch.cat([oc, mc], 1).permute(0, 2, 3, 1).contiguous()
        cols = torch.full((B * Ho * Wo, K * C), 7.0, device="cuda")
        call("vd3d_deform_im2col_nhwc", xn.data_ptr(), B, H, W, C, C, 0, om.data_ptr(), om.shape[3], 0,
             om.data_ptr() if v2 else None, om.shape[3], 2 * K * dg, 0, k, k, s, p, d, dg, cols.data_ptr(), None, K * C, E._stream())
        torch.cuda.synchronize()
        check(cols.view(B, Ho, Wo, K * C), r["cols"], COL_N * U * r["abs_cols"] + 1e-300, f"columns {'v2' if v2 else 'v1'} {case} {family}")


# ---- taps exactly on the validity boundary read nothing -------------------------------------------------------------------------------
def test_boundary_taps_read_nothing(monkeypatch):
    """Every tap sits exactly at -1 or at H / W (dcn_cases.boundary_offsets), so none is valid and each output is its bias, exactly, even
    though row 0 and column 0 of the image are NaN: a tap at exactly -1 must be skipped like the reference skips it, not evaluated with a
    zero bilinear weight (0 * NaN would reach the output).  (Splitting the NaN image into fp16 planes trips the library's sticky fp16-range
    flag; it is cleared at the end so later work in the process does not report it.)"""
    try:
        _boundary_cases(monkeypatch)
    finally:
        E.fp16_range_overflowed(reset=True)


def _boundary_cases(monkeypatch):
    def image(B, C, H, W):
        x = torch.randn(B, C, H, W, generator=torch.Generator().manual_seed(H))
        x[:, :, 0, :] = float("nan")
        x[:, :, :, 0] = float("nan")
        return x
    for (B, C, H, W, Co, k, s, p, d, dg, variants) in ((2, 64, 13, 21, 48, 3, 1, 1, 1, 1, [("1", "1"), ("1", "0"), ("0", "1")]),
                                                       (1, 64, 11, 17, 24, 3, 2, 1, 1, 1, [("1", "0"), ("0", "0")]),
                                                       (1, 32, 9, 12, 16, 5, 1, 2, 1, 2, [("0", "1")])):
        off = dc.boundary_offsets(B, H, W, k, k, s, p, d, dg)
        got, want, bound, layer = layer_case(B, C, H, W, Co, k, s, p, d, dg, None, relu=False, seed=7, monkeypatch=monkeypatch,
                                             variants=variants, x=image(B, C, H, W), off=off, res_on=False)
        assert torch.equal(got.double(), want), "a boundary tap contributed"
    # ops API (fp32 columns + 3xTF32 GEMM) and the column tensor
    B, C, H, W, Co, k, s, p, d, dg = 1, 8, 9, 11, 5, 3, 1, 1, 1, 2
    x = image(B, C, H, W).cuda()
    w = torch.randn(Co, C, k, k, device="cuda")
    bias = torch.randn(Co, device="cuda")
    off = dc.boundary_offsets(B, H, W, k, k, s, p, d, dg).cuda()
    mask = torch.rand(B, k * k * dg, *off.shape[2:], device="cuda")
    out = torch.empty(B, Co, *off.shape[2:], device="cuda")
    e = x.new_empty(0)
    dcn.modulated_deform_conv_forward(x, w, bias, e, off, mask, out, e, k, k, s, s, p, p, d, d, 1, dg, True)
    torch.cuda.synchronize()
    assert torch.equal(out, bias[None, :, None, None].expand_as(out))
    assert dcn.deform_conv_forward(x, w, off, out, e, e, k, k, s, s, p, p, d, d, 1, dg, B) == 1
    torch.cuda.synchronize()
    assert torch.equal(out, torch.zeros_like(out))


# ---- backward through the ops API ------------------------------------------------------------------------------------------------------
# B, C, H, W, Cout, k, stride, pad, dil, dg: K = 1 / 9 / 25 / 49, stride 2, dilation 2, C / dg = 4, B*Ho*Wo not a multiple of 16
BWD = [(1, 4, 9, 11, 5, 1, 1, 0, 1, 1), (2, 8, 10, 13, 6, 3, 1, 1, 1, 2), (1, 16, 12, 17, 4, 5, 2, 2, 1, 4), (1, 8, 11, 13, 3, 7, 1, 3, 1, 2),
       (2, 4, 13, 10, 4, 3, 1, 2, 2, 1)]


@pytest.mark.parametrize("family", dc.FAMILIES)
@pytest.mark.parametrize("case", BWD)
def test_ops_backward_on_families(case, family):
    B, C, H, W, Co, k, s, p, d, dg = case
    Ho, Wo = dc.out_hw(H, W, k, k, s, p, d)
    assert (B * Ho * Wo) % 16 != 0 and C // dg == 4
    x, w, b, off, mask = ops_inputs(case, family, 100 + BWD.index(case))
    gout = torch.randn(B, Co, Ho, Wo, generator=torch.Generator().manual_seed(9))
    xc, wc, bc, oc, mc, gc = x.cuda(), w.cuda(), b.cuda(), off.cuda(), mask.cuda(), gout.cuda()
    e = xc.new_empty(0)
    npix, cq = B * Ho * Wo, C // dg // 4

    def bounds(r):
        return dict(grad_input=(4 + Co + r["count_input"]) * U * r["abs_grad_input"],
                    grad_offset=(Co + 10 + cq) * U * r["abs_grad_offset"],
                    grad_mask=(Co + 10 + cq) * U * r["abs_grad_mask"] if r["abs_grad_mask"] is not None else None,
                    grad_weight=(COL_N + npix + 2) * U * r["abs_grad_weight"],
                    grad_bias=(npix + 1) * U * r["abs_grad_bias"])

    def compare(got, r, bd, tag, factor=1.0):
        for name, t in got.items():
            check(t, factor * r[name], factor * bd[name] + 1e-300, f"{tag} {name} {case} {family}")
        if "grad_offset" in got:
            assert bool((got["grad_offset"][r["edge"].cuda()] == 0.0).all()), "coordinate gradient at exactly -1 must be 0.0"

    # ---- DCNv2 ----
    r = dc.backward(xc, oc, mc, wc, gc, s, p, d, dg)
    bd = bounds(r)
    gi, gw, gb = torch.zeros_like(xc), torch.zeros_like(wc), torch.zeros_like(bc)
    go, gm = torch.full_like(oc, 3.0), torch.full_like(mc, 3.0)
    dcn.modulated_deform_conv_backward(xc, wc, bc, e, oc, mc, e, gi, gw, gb, go, gm, gc, k, k, s, s, p, p, d, d, 1, dg, True)
    torch.cuda.synchronize()
    compare(dict(grad_input=gi, grad_offset=go, grad_mask=gm, grad_weight=gw, grad_bias=gb), r, bd, "v2")
    # grad_input / grad_weight / grad_bias are accumulated into, grad_offset / grad_mask assigned
    dcn.modulated_deform_conv_backward(xc, wc, bc, e, oc, mc, e, gi, gw, gb, go, gm, gc, k, k, s, s, p, p, d, d, 1, dg, True)
    torch.cuda.synchronize()
    compare(dict(grad_input=gi, grad_weight=gw, grad_bias=gb), r, bd, "v2 x2", 2.0)
    compare(dict(grad_offset=go, grad_mask=gm), r, bd, "v2 again")
    # ---- DCNv1 ----
    r = dc.backward(xc, oc, None, wc, gc, s, p, d, dg)
    bd = bounds(r)
    gi, go, gw = torch.zeros_like(xc), torch.full_like(oc, 3.0), torch.zeros_like(wc)
    assert dcn.deform_conv_backward_input(xc, oc, gc, gi, go, wc, e, k, k, s, s, p, p, d, d, 1, dg, B) == 1
    assert dcn.deform_conv_backward_parameters(xc, oc, gc, gw, e, e, k, k, s, s, p, p, d, d, 1, dg, 0.5, B) == 1
    torch.cuda.synchronize()
    compare(dict(grad_input=gi, grad_offset=go), r, bd, "v1")
    compare(dict(grad_weight=gw), r, bd, "v1 scale 0.5", 0.5)
