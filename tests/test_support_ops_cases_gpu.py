"""-m gpu: the fp32 support kernels on the constructed cases of tests/support_ops_cases.py, against float64.

Each kernel runs through the C ABI into a channel slice of a buffer filled with SENTINEL, reading its inputs from slices whose neighbouring
channels hold SENTINEL too; every test asserts the neighbouring channels (and planes) are untouched.

Checks:
  * exact operands (integers and multiples of 1/8, every partial sum exact in float32): the device equals float64 bit for bit;
  * random normals: |device - float64| <= bound per element, the assertion is on max |err| / bound <= 1 and the ratio is printed:
      SIMT conv          gamma(K + 2) * (conv(|x|, |w|) + |b| + |r|)     K fmas, the bias add, the residual add
      avgpool2           gamma(3) * sum|x| / 4                          three adds; the division by 4 is exact
      dwconv3x3          gamma(10) * (conv(|x|, |w|) + |b|)             9 fmas, the bias add
      dw_convtranspose   gamma(5) * (convT(|x|, |w|) + |a|)             at most 2 x 2 taps, the addend
      LookGround         support_ops_cases.lg_bound                     weights and sum, plus the sampling-position slack
  * layout converters, max pools, channel copy and the splitters: bit for bit.
"""
import numpy as np
import pytest
import torch

import support_ops_cases as sc
from visualdet3d_b200 import engine as E
from visualdet3d_b200._lib import call

pytestmark = pytest.mark.gpu
SENT = sc.SENTINEL


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def nchw(t):
    return t.permute(0, 3, 1, 2).contiguous()


def slot(data_nchw, cs, co, extra_images=0):
    """[B, H, W, cs] device buffer of SENTINEL with data_nchw [B, C, H, W] in channels [co, co + C) (extra_images: more SENTINEL images
    after the last)"""
    B, C, H, W = data_nchw.shape
    buf = torch.full((B + extra_images, H, W, cs), SENT, device="cuda")
    buf[:B, ..., co:co + C] = nhwc(data_nchw).cuda()
    return buf


def assert_outside_untouched(buf, co, C, what):
    assert bool((buf[..., :co] == SENT).all()) and bool((buf[..., co + C:] == SENT).all()), f"{what}: neighbouring channels written"


def check_bound(got, want, bound, what):
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    r = sc.err_ratio(got, want, bound)
    print(f"  {what}: max |err| / bound = {r:.3g}")
    assert r <= 1.0, (what, r)
    return r


# ---- SIMT conv ---------------------------------------------------------------------------------------------------------------------------
def run_simt(c, x, w, b, r, in_cs=None, in_co=None, misalign=False):
    """vd3d_conv2d_nhwc into channels [4, 4 + Cout) of a Cout + 8 wide buffer; residual from channels [8, 8 + Cout) of a Cout + 12 wide one.
    Returns (out [B, Cout, Ho, Wo] float32 on the CPU, the output buffer)."""
    Ho, Wo, _, _ = sc.conv_dims(c)
    in_cs = c.in_cs if in_cs is None else in_cs
    in_co = c.in_co if in_co is None else in_co
    xb = slot(x, in_cs, in_co)
    if misalign:                                   # same values, base pointer 4 bytes past a 16-byte boundary
        flat = torch.full((xb.numel() + 1,), SENT, device="cuda")
        flat[1:] = xb.reshape(-1)
        xb = flat[1:].view(xb.shape)
        assert xb.data_ptr() % 16 == 4
    wk = sc.pack_conv_weight(w).cuda()
    bd = b.cuda() if b is not None else None
    rb = slot(r, c.Cout + 12, 8) if r is not None else None
    ob = torch.full((c.B, Ho, Wo, c.Cout + 8), SENT, device="cuda")
    call("vd3d_conv2d_nhwc", xb.data_ptr(), c.B, c.H, c.W, c.Cin, in_cs, in_co, wk.data_ptr(), bd.data_ptr() if bd is not None else None,
         c.KH, c.KW, c.stride, c.pad, c.dil, rb.data_ptr() if rb is not None else None, c.Cout + 12, 8,
         ob.data_ptr(), c.Cout, c.Cout + 8, 4, 1 if c.relu else 0, None)
    torch.cuda.synchronize()
    assert_outside_untouched(ob, 4, c.Cout, c.name)
    if rb is not None:
        assert_outside_untouched(rb, 8, c.Cout, c.name + " residual")
    return nchw(ob[..., 4:4 + c.Cout]).cpu(), ob


@pytest.mark.parametrize("c", sc.CONV_CASES, ids=lambda c: c.name)
def test_simt_conv_exact(c):
    x, w, b, r = sc.conv_operands(c, "exact", 0)
    got, _ = run_simt(c, x, w, b, r)
    want, _ = sc.conv_ref(x, w, b, r, c.stride, c.pad, c.dil, c.relu)
    assert torch.equal(got.double(), want), f"{c.name}: max |err| = {float((got.double() - want).abs().max())}"


@pytest.mark.parametrize("c", sc.CONV_CASES, ids=lambda c: c.name)
def test_simt_conv_within_bound(c):
    x, w, b, r = sc.conv_operands(c, "normal", 1)
    got, _ = run_simt(c, x, w, b, r)
    want, S = sc.conv_ref(x, w, b, r, c.stride, c.pad, c.dil, c.relu)
    check_bound(got, want, sc.gamma(sc.conv_dims(c)[3] + 2) * S, f"simt conv {c.name}")


@pytest.mark.parametrize("p", sc.PAIR_CASES, ids=lambda p: p[0])
def test_simt_scalar_and_vector_gathers_are_bit_identical(p):
    name, B, Cin, H, W, Cout, KH, KW, s, pad, d, in_cs = p
    c = sc.ConvCase(name, B, Cin, H, W, Cout, KH, KW, s, pad, d, True, True, True, in_cs, 0, None)
    x, w, b, r = sc.conv_operands(c, "normal", 2)
    vec, _ = run_simt(c, x, w, b, r, in_co=sc.PAIR_IN_CO[0])
    scal, _ = run_simt(c, x, w, b, r, in_co=sc.PAIR_IN_CO[1])
    unal, _ = run_simt(c, x, w, b, r, in_co=sc.PAIR_IN_CO[0], misalign=True)
    assert torch.equal(vec.view(torch.int32), scal.view(torch.int32)), f"{name}: scalar gather differs from the float4 gather"
    assert torch.equal(vec.view(torch.int32), unal.view(torch.int32)), f"{name}: unaligned base pointer differs"
    want, S = sc.conv_ref(x, w, b, r, s, pad, d, True)
    check_bound(vec, want, sc.gamma(KH * KW * Cin + 2) * S, f"simt conv {name}")


# ---- layout converters -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", sc.LAYOUT_C)
@pytest.mark.parametrize("hw", sc.LAYOUT_HW, ids=lambda hw: f"{hw[0]}x{hw[1]}")
def test_layout_converters_bit_exact(C, hw):
    H, W = hw
    B, co, cs = 2, sc.LAYOUT_CO, C + 5
    g = torch.Generator().manual_seed(C * 100 + H)
    x = torch.randn(B, C, H, W, generator=g)
    # NCHW -> NHWC into channels [co, co + C)
    ob = torch.full((B, H, W, cs), SENT, device="cuda")
    xd = x.cuda()
    call("vd3d_nchw_to_nhwc", xd.data_ptr(), ob.data_ptr(), B, C, H, W, cs, co, None)
    assert torch.equal(ob[..., co:co + C].cpu(), x.permute(0, 2, 3, 1)), sc.nchw_to_nhwc_kernel(C)
    assert_outside_untouched(ob, co, C, "nchw_to_nhwc")
    # NHWC channels [co, co + C) -> NCHW
    ib = slot(x, cs, co)
    out = torch.full((B, C, H, W), SENT, device="cuda")
    call("vd3d_nhwc_to_nchw", ib.data_ptr(), out.data_ptr(), B, C, H, W, cs, co, None)
    assert torch.equal(out.cpu(), x)


# ---- pools -------------------------------------------------------------------------------------------------------------------------------
def run_pool(entry, x, Ho, Wo, in_cs=16, in_co=4, out_cs=20, out_co=8):
    B, C, H, W = x.shape
    xb = slot(x, in_cs, in_co)
    ob = torch.full((B, Ho, Wo, out_cs), SENT, device="cuda")
    call(entry, xb.data_ptr(), B, H, W, C, in_cs, in_co, ob.data_ptr(), out_cs, out_co, None)
    torch.cuda.synchronize()
    assert_outside_untouched(ob, out_co, C, entry)
    return nchw(ob[..., out_co:out_co + C]).cpu()


@pytest.mark.parametrize("kind", sc.POOL_KINDS)
@pytest.mark.parametrize("hw", sc.MAXPOOL3_HW, ids=lambda hw: f"{hw[0]}x{hw[1]}")
def test_maxpool3x3s2_bit_exact(hw, kind):
    H, W = hw
    x = sc.pool_input(2, 8, H, W, kind, H * 10 + W)
    got = run_pool("vd3d_maxpool3x3s2_nhwc", x, *sc.maxpool3_out_hw(H, W))
    assert torch.equal(got.double(), sc.maxpool3_ref(x))


@pytest.mark.parametrize("kind", sc.POOL_KINDS)
@pytest.mark.parametrize("hw", sc.MAXPOOL2_HW, ids=lambda hw: f"{hw[0]}x{hw[1]}")
def test_maxpool2x2s2_bit_exact(hw, kind):
    H, W = hw
    x = sc.pool_input(2, 8, H, W, kind, H * 10 + W)
    got = run_pool("vd3d_maxpool2x2s2_nhwc", x, H // 2, W // 2)
    assert torch.equal(got.double(), sc.maxpool2_ref(x))


@pytest.mark.parametrize("hw", sc.AVGPOOL_HW, ids=lambda hw: f"{hw[0]}x{hw[1]}")
def test_avgpool2(hw):
    H, W = hw
    xd = sc.pool_input(2, 12, H, W, "dyadic", H)
    got = run_pool("vd3d_avgpool2_nhwc", xd, H // 2, W // 2)
    assert torch.equal(got.double(), sc.avgpool2_ref(xd)[0])
    xn = sc.pool_input(2, 12, H, W, "normal", H + 1)
    got = run_pool("vd3d_avgpool2_nhwc", xn, H // 2, W // 2)
    want, S = sc.avgpool2_ref(xn)
    check_bound(got, want, sc.gamma(3) * S, f"avgpool2 {H}x{W}")


@pytest.mark.parametrize("case", sc.COPY_CASES, ids=lambda c: f"C{c[1]}")
def test_copy_channels_bit_exact(case):
    (B, H, W), C, in_cs, in_co, out_cs, out_co = case
    x = torch.randn(B, C, H, W, generator=torch.Generator().manual_seed(C))
    xb = slot(x, in_cs, in_co)
    ob = torch.full((B, H, W, out_cs), SENT, device="cuda")
    call("vd3d_copy_channels_nhwc", xb.data_ptr(), B * H * W, C, in_cs, in_co, ob.data_ptr(), out_cs, out_co, None)
    assert torch.equal(ob[..., out_co:out_co + C].cpu(), nhwc(x))
    assert_outside_untouched(ob, out_co, C, "copy_channels")


# ---- depthwise ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ("exact", "normal"))
@pytest.mark.parametrize("case", sc.DWCONV_CASES, ids=lambda c: "B{}_{}x{}_C{}_bias{}_relu{}".format(*c))
def test_dwconv3x3(case, kind):
    B, H, W, C, bias, relu = case
    x, w, b = sc.dwconv_operands(B, H, W, C, bias, kind, C + H)
    in_cs, in_co, out_cs, out_co = C + 8, 4, C + 12, 8
    xb = slot(x, in_cs, in_co)
    wk = w.reshape(C, 9).t().contiguous().cuda()
    bd = b.cuda() if b is not None else None
    ob = torch.full((B, H, W, out_cs), SENT, device="cuda")
    call("vd3d_dwconv3x3_nhwc", xb.data_ptr(), B, H, W, C, in_cs, in_co, wk.data_ptr(), bd.data_ptr() if bd is not None else None,
         ob.data_ptr(), out_cs, out_co, 1 if relu else 0, None)
    got = nchw(ob[..., out_co:out_co + C]).cpu()
    assert_outside_untouched(ob, out_co, C, "dwconv3x3")
    want, S = sc.dwconv_ref(x, w, b, relu)
    if kind == "exact":
        assert torch.equal(got.double(), want)
    else:
        check_bound(got, want, sc.gamma(10) * S, f"dwconv3x3 {case}")


@pytest.mark.parametrize("kind", ("exact", "normal"))
@pytest.mark.parametrize("case", sc.DWT_CASES, ids=lambda c: "B{}_{}x{}_C{}_f{}_add{}".format(*c))
def test_dw_convtranspose(case, kind):
    B, H, W, C, f, addend = case
    x, w, a = sc.dwt_operands(B, H, W, C, f, addend, kind, 7 * f + H)
    in_cs, in_co, add_cs, add_co, out_cs, out_co = C + 4, 4, C + 8, 8, C + 8, 4
    xb = slot(x, in_cs, in_co)
    wk = w.reshape(C, -1).t().contiguous().cuda()
    ab = slot(a, add_cs, add_co) if a is not None else None
    ob = torch.full((B, H * f, W * f, out_cs), SENT, device="cuda")
    call("vd3d_dw_convtranspose_nhwc", xb.data_ptr(), B, H, W, C, in_cs, in_co, wk.data_ptr(), f,
         ab.data_ptr() if ab is not None else None, add_cs, add_co, ob.data_ptr(), out_cs, out_co, None)
    got = nchw(ob[..., out_co:out_co + C]).cpu()
    assert_outside_untouched(ob, out_co, C, "dw_convtranspose")
    want, S = sc.dwt_ref(x, w, a, f)
    if kind == "exact":
        assert torch.equal(got.double(), want)
    else:
        check_bound(got, want, sc.gamma(5) * S, f"dw_convtranspose {case}")


# ---- LookGround ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", sc.LG_CASES, ids=lambda c: c.name)
def test_look_ground_sample(c):
    x, d, P2 = sc.lg_inputs(c, 0)
    # one guard image of +inf after the last: a corner the kernel must skip (x1 = W, y1 = H) but reads anyway turns 0 * inf into NaN
    xb = slot(x, c.x_cs, c.x_co, extra_images=1)
    xb[c.B:] = float("inf")
    db = slot(d[:, None], c.d_cs, c.d_co)
    ocs = sc.lg_out_cs(c)
    ob = torch.full((c.B, c.H, c.W, ocs), SENT, device="cuda")
    lb = torch.full((c.B, c.H, c.W, ocs), SENT, device="cuda")
    P2d = P2.contiguous().cuda()
    call("vd3d_look_ground_sample", xb.data_ptr(), c.B, c.H, c.W, c.C, c.x_cs, c.x_co, db.data_ptr(), c.d_cs, c.d_co, P2d.data_ptr(),
         sc.LG_BASELINE, c.elev, ob.data_ptr(), lb.data_ptr(), ocs, None)
    torch.cuda.synchronize()
    for buf, nm in ((ob, "out"), (lb, "lo")):
        assert bool((buf[..., c.C + 1:] == SENT).all()), f"{nm}: channels beyond C + 1 written"
    got = ob[..., :c.C + 1]
    # the tf32 companion is exactly value - trunc13(value)
    assert torch.equal(lb[..., :c.C + 1], got - sc.trunc13(got))
    want, S, M = sc.lg_ref(x, d, P2, c.elev)
    got = nchw(got).cpu()
    if c.name.startswith("integer_grid"):
        assert torch.equal(got[:, :c.C], x)                     # every tap on an integer: the sampler is a copy
    check_bound(got, want, sc.lg_bound(S, M, c.H, c.W), f"look_ground {c.name}")


# ---- splitters ---------------------------------------------------------------------------------------------------------------------------
def run_split_h16(vals, C=12, cs=20, co=4):
    t = sc.to_channels(vals, C)                                  # [npix, C]
    npix = t.shape[0]
    xb = torch.full((npix, cs), SENT, device="cuda")
    xb[:, co:co + C] = t.cuda()
    planes = torch.full((2, npix, cs), 7.0, device="cuda", dtype=torch.float16)
    call("vd3d_split_h16_nhwc", xb.data_ptr(), planes[0].data_ptr(), planes[1].data_ptr(), npix, C, cs, co, None)
    torch.cuda.synchronize()
    assert bool((planes[..., :co] == 7.0).all()) and bool((planes[..., co + C:] == 7.0).all()), "split_h16: neighbouring channels written"
    return t, planes[0, :, co:co + C].cpu(), planes[1, :, co:co + C].cpu()


def test_split_h16_ties_subnormals_and_range_edge():
    E.fp16_range_overflowed(reset=True)
    g = torch.Generator().manual_seed(0)
    vals = sc.fp16_ties() + sc.fp16_specials() + (torch.randn(200, generator=g) * 100).tolist()
    t, hi, lo = run_split_h16(vals)
    rh, rl = sc.split_h16_ref(t)
    assert torch.equal(hi.view(torch.int16), rh.view(torch.int16)), "hi plane differs from t.half()"
    assert torch.equal(lo.view(torch.int16), rl.view(torch.int16)), "lo plane differs from (t - hi).half()"
    assert not E.fp16_range_overflowed(reset=True), "range flag raised below 65520"


def test_split_h16_overflow_raises_and_clears_the_flag():
    E.fp16_range_overflowed(reset=True)
    t, hi, lo = run_split_h16(sc.fp16_overflows() + [1.0, -2.5])
    rh, rl = sc.split_h16_ref(t)
    assert torch.equal(hi.view(torch.int16), rh.view(torch.int16)) and torch.equal(lo.view(torch.int16), rl.view(torch.int16))
    assert torch.isinf(hi[0, :len(sc.fp16_overflows())].float()).all()
    assert E.fp16_range_overflowed(reset=True), "range flag not raised at |v| >= 65520"
    assert not E.fp16_range_overflowed(reset=True), "range flag not cleared on read"


def test_split_lo_is_value_minus_trunc13():
    g = torch.Generator().manual_seed(1)
    vals = (torch.randn(300, generator=g) * torch.exp2(torch.randint(-30, 30, (300,), generator=g).float())).tolist()
    vals += sc.fp16_specials() + sc.fp16_overflows() + [2.0 ** -140, -(2.0 ** -130), 2.0 ** 120]
    C, cs, co = 12, 24, 8
    t = sc.to_channels(vals, C)
    npix = t.shape[0]
    xb = torch.full((npix, cs), SENT, device="cuda")
    xb[:, co:co + C] = t.cuda()
    lo = torch.full((npix, cs), SENT, device="cuda")
    call("vd3d_split_lo_nhwc", xb.data_ptr(), lo.data_ptr(), npix, C, cs, co, None)
    torch.cuda.synchronize()
    assert torch.equal(lo[:, co:co + C].cpu().view(torch.int32), (t - sc.trunc13(t)).view(torch.int32))
    assert_outside_untouched(lo, co, C, "split_lo")
