"""-m gpu: the tensor-core conv engine on the constructed cases of tests/tc_conv_cases.py, against float64.

The C entries are called directly with ctypes arrays, so the fp16 planes and every pointer are the test's own:
  * input planes live in a channel slice of a wider buffer whose other channels, and one extra image after the B the kernel is told about,
    hold fp16 +inf: a read outside the slice (or a padding tap that is not zero fill) turns into inf / NaN in the output;
  * output fp32 and both output planes are pre-filled with a sentinel outside the channel slice, in one extra trailing image and (multi-level
    launches) in the gaps between levels, and must be unchanged afterwards;
  * exact operands, one family per plane product ((a) x_hi w_hi, (b) x_lo w_hi, (c) x_hi w_lo, (d) x_lo w_lo only, which the engine drops):
    the fp32 output and both output planes equal float64 bit for bit; (b) with passes = 2 (A_lo * W_hi dropped) gives exactly bias + residual;
  * random normals: max |err| / bound <= 1 per element with the bound of tc_conv_cases.tc16_bound / tf32_bound; the ratio is printed per row
    and the largest per family at the end of the module;
  * the fp16 range flag at tile edges, and bit-identity wherever the engine claims it (every tile width, VD3D_ROW64, VD3D_TC_TILE_IN_RING,
    v8 on / off, multi-level against per-level launches).
"""
import contextlib
import ctypes
import os

import pytest
import torch

import tc_conv_cases as tc
from visualdet3d_b200 import engine as E
from visualdet3d_b200._lib import call

pytestmark = pytest.mark.gpu

INF = float("inf")
SENT32 = -777.25
SENT16 = -1234.0
RATIOS = {}


@pytest.fixture(scope="module", autouse=True)
def ratio_summary():
    yield
    for fam, (r, name) in sorted(RATIOS.items()):
        print(f"  max |err| / bound, {fam}: {r:.3g} ({name})")


def note_ratio(fam, name, r):
    print(f"  {fam} {name}: max |err| / bound = {r:.3g}")
    if r > RATIOS.get(fam, (-1.0, ""))[0]:
        RATIOS[fam] = (r, name)
    assert r <= 1.0, (fam, name, r)


@contextlib.contextmanager
def engine_env(env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def P(ptrs):
    return (ctypes.c_void_p * len(ptrs))(*ptrs)


def I(vals):
    return (ctypes.c_int * len(vals))(*vals)


def nhwc(t):
    return t.permute(0, 2, 3, 1)


def nchw(t):
    return t.permute(0, 3, 1, 2).contiguous()


def slot(data, cs, co, fill, dtype):
    """[B + 1, H, W, cs] device buffer of `fill` with data [B, C, H, W] in channels [co, co + C) of the first B images"""
    B, C, H, W = data.shape
    buf = torch.full((B + 1, H, W, cs), fill, dtype=dtype, device="cuda")
    buf[:B, ..., co:co + C] = nhwc(data).to(dtype).cuda()
    return buf


def bias_slot(b, mis):
    """bias in a larger +inf buffer: 16 bytes past a 32-byte boundary (mis) or 32-byte aligned, with slack after Cout"""
    off = 4 if mis else 8
    buf = torch.full((b.numel() + 16,), INF, device="cuda")
    buf[off:off + b.numel()] = b.float().cuda()
    v = buf[off:off + b.numel()]
    assert v.data_ptr() % 32 == (16 if mis else 0)
    return buf, v


class Outputs:
    """output forms of one launch: [npix, cs] sentinel buffers (fp32 and / or fp16 planes) and the pixel ranges the kernel may write"""

    def __init__(self, npix, cs, f32, planes):
        self.f32 = torch.full((npix, cs), SENT32, device="cuda") if f32 else None
        self.hi = torch.full((npix, cs), SENT16, dtype=torch.float16, device="cuda") if planes else None
        self.lo = torch.full((npix, cs), SENT16, dtype=torch.float16, device="cuda") if planes else None

    def ptrs(self, t, pix_offs, cs, esize):
        return None if t is None else P([t.data_ptr() + o * cs * esize for o in pix_offs])

    def check_untouched(self, regions, co, C, what):
        """regions: (first pixel, pixel count) the kernel writes, channels [co, co + C)"""
        for t, s in ((self.f32, SENT32), (self.hi, SENT16), (self.lo, SENT16)):
            if t is None:
                continue
            m = torch.ones(t.shape, dtype=torch.bool, device="cuda")
            for p0, n in regions:
                m[p0:p0 + n, co:co + C] = False
            assert bool((t[m] == s).all()), f"{what}: the kernel wrote outside its output slice"

    def get(self, p0, B, Ho, Wo, co, C):
        """NCHW (f32, hi, lo) of one level on the CPU (None for a form not written)"""
        ex = lambda t: None if t is None else nchw(t[p0:p0 + B * Ho * Wo, co:co + C].reshape(B, Ho, Wo, C)).cpu()
        return ex(self.f32), ex(self.hi), ex(self.lo)


def flag_clear():
    E.fp16_range_overflowed()


# ---- vd3d_conv2d_tc16 ----------------------------------------------------------------------------------------------------------------------
def run_tc16(B, Cin, in_cs, in_co, levels, Cout, out_cs, out_co, KH, KW, stride, pad, dil, w_planes, osc, b, bias_mis, res, res_kind, outf, relu,
             bn, passes=3, env=(), what=""):
    """One vd3d_conv2d_tc16 launch over len(levels) levels.  levels[l] = (x_hi, x_lo) CPU fp16 [B, Cin, H, W]; res[l]: float64 NCHW residual
    (half the output size for res_kind "up") or None.  Returns the per-level NCHW (f32, hi, lo) on the CPU."""
    L = len(levels)
    hws = [(xh.shape[2], xh.shape[3]) for xh, _ in levels]
    ohws = [tc.out_hw(H, W, KH, KW, stride, pad, dil) for H, W in hws]
    xb = [(slot(xh, in_cs, in_co, INF, torch.float16), slot(xl, in_cs, in_co, INF, torch.float16)) for xh, xl in levels]
    whi, wlo = w_planes[0].cuda(), w_planes[1].cuda()
    bbuf, bias = bias_slot(b, bias_mis)
    offs, npix = tc.level_offsets(B, ohws) if L > 1 else ([0], B * ohws[0][0] * ohws[0][1] + ohws[0][0] * ohws[0][1])
    out = Outputs(npix, out_cs, outf in ("f32", "both"), outf in ("planes", "both"))
    r32 = rhi = rlo = None
    rH = rW = None
    keep = []
    if res_kind != "none":
        rhws = [(r.shape[2], r.shape[3]) for r in res]
        roffs, rpix = tc.level_offsets(B, rhws)
        if res_kind == "planes":
            rhi_t = torch.full((rpix, out_cs), INF, dtype=torch.float16, device="cuda")
            rlo_t = torch.full((rpix, out_cs), INF, dtype=torch.float16, device="cuda")
            for r, o in zip(res, roffs):
                h, lo_ = tc.split16(r)
                rhi_t[o:o + r.numel() // Cout, out_co:out_co + Cout] = nhwc(h).reshape(-1, Cout).cuda()
                rlo_t[o:o + r.numel() // Cout, out_co:out_co + Cout] = nhwc(lo_).reshape(-1, Cout).cuda()
            keep += [rhi_t, rlo_t]
            rhi = P([rhi_t.data_ptr() + o * out_cs * 2 for o in roffs])
            rlo = P([rlo_t.data_ptr() + o * out_cs * 2 for o in roffs])
        else:
            r_t = torch.full((rpix, out_cs), INF, device="cuda")
            for r, o in zip(res, roffs):
                r_t[o:o + r.numel() // Cout, out_co:out_co + Cout] = nhwc(r).reshape(-1, Cout).float().cuda()
            keep.append(r_t)
            r32 = P([r_t.data_ptr() + o * out_cs * 4 for o in roffs])
            if res_kind == "up":
                rH, rW = I([h for h, _ in rhws]), I([w for _, w in rhws])
    with engine_env(dict(env)):
        call("vd3d_conv2d_tc16", L, P([h.data_ptr() for h, _ in xb]), P([l.data_ptr() for _, l in xb]), I([h for h, _ in hws]), I([w for _, w in hws]),
             B, Cin, in_cs, in_co, whi.data_ptr(), wlo.data_ptr(), osc, bias.data_ptr(), KH, KW, pad, dil, stride,
             r32, rhi, rlo, rH, rW, out_cs if res_kind != "none" else 0, out_co if res_kind != "none" else 0,
             out.ptrs(out.f32, offs, out_cs, 4), out.ptrs(out.hi, offs, out_cs, 2), out.ptrs(out.lo, offs, out_cs, 2),
             Cout, out_cs, out_co, 1 if relu else 0, passes, bn, None)
    torch.cuda.synchronize()
    out.check_untouched([(o, B * h * w) for o, (h, w) in zip(offs, ohws)], out_co, Cout, what)
    assert bool(torch.isinf(bbuf[:4 if bias_mis else 8]).all()) and bool(torch.isinf(bbuf[(4 if bias_mis else 8) + Cout:]).all())
    return [out.get(o, B, h, w, out_co, Cout) for o, (h, w) in zip(offs, ohws)]


def run_conv(c, x_planes, w_planes, osc, b, r, passes=3, env=None, bias_mis=None):
    env = dict(c.env) if env is None else env
    return run_tc16(c.B, c.Cin, c.in_cs, c.in_co, [x_planes], c.Cout, c.out_cs, c.out_co, c.KH, c.KW, c.stride, c.pad, c.dil, w_planes, osc, b,
                    c.bias_mis if bias_mis is None else bias_mis, [r] if r is not None else None, c.res, c.outf, c.relu, c.bn, passes, env.items(),
                    c.name)[0]


def assert_exact(got, want, what):
    """every written form equals the float64 value bit for bit (fp32, and the planes hi = rn16(v), lo = rn16(v - hi))"""
    f32, hi, lo = got
    w32 = want.float()
    assert torch.equal(w32.double(), want), f"{what}: the reference is not exact in float32"
    if f32 is not None:
        d = (f32.double() - want).abs()
        assert torch.equal(f32, w32), f"{what}: fp32 output differs from float64 (max |err| {float(d.nan_to_num(INF).max())}, " \
                                      f"{int((d != 0).sum())} elements)"
    if hi is not None:
        wh = w32.half()
        assert torch.equal(hi, wh), f"{what}: hi plane differs from float64"
        assert torch.equal(lo, (w32 - wh.float()).half()), f"{what}: lo plane differs from float64"


def assert_same_bits(a, b, what):
    for x, y in zip(a, b):
        assert (x is None) == (y is None)
        if x is not None:
            assert torch.equal(x.view(torch.int16) if x.dtype == torch.float16 else x.view(torch.int32),
                               y.view(torch.int16) if y.dtype == torch.float16 else y.view(torch.int32)), f"{what}: not bit-identical"


def plane_families(xh, wh):
    """(x_hi, x_lo, w_hi, w_lo) of the four exact families from exact x and scaled weight planes with lo = 0"""
    zx, zw = torch.zeros_like(xh), torch.zeros_like(wh)
    return {"a": (xh, zx, wh, zw), "b": (zx, xh, wh, zw), "c": (xh, zx, zw, wh), "d": (zx, xh, zw, wh)}


def res_shape(c, B, Ho, Wo):
    if c.res == "none":
        return None
    return (B, c.Cout, Ho // 2, Wo // 2) if c.res == "up" else (B, c.Cout, Ho, Wo)


def exact_conv_setup(c, seed):
    Ho, Wo = tc.out_hw(c.H, c.W, c.KH, c.KW, c.stride, c.pad, c.dil)
    x, w, b, r = tc.exact_operands(c.B, c.Cin, c.H, c.W, c.Cout, c.KH, c.KW, res_shape(c, c.B, Ho, Wo), seed)
    cin64 = tc.cdiv(c.Cin, 64) * 64
    whi, wlo, osc = E.fp16_split_scaled(tc.pack_weight(w, cin64))
    assert osc == 2.0 ** -14 and not bool(wlo.float().any())
    return x, w, b, r, whi, osc


@pytest.mark.parametrize("c", tc.CONV_CASES, ids=lambda c: c.name)
def test_conv_plane_products_exact(c):
    x, w, b, r, whi, osc = exact_conv_setup(c, 10)
    want, _ = tc.conv_ref(x, w, b, r, c.stride, c.pad, c.dil, c.relu, c.res == "up")
    bias_res = tc.epilogue_ref(torch.zeros_like(want), b, r, c.relu, c.res == "up")
    for fam, (xh, xl, wh, wl) in plane_families(x.half(), whi).items():
        got = run_conv(c, (xh, xl), (wh, wl), osc, b, r)
        assert_exact(got, bias_res if fam == "d" else want, f"{c.name} family {fam}")
    if c.res != "planes":
        fam_b = plane_families(x.half(), whi)["b"]
        got = run_conv(c, fam_b[:2], fam_b[2:], osc, b, r, passes=2)
        assert_exact(got, bias_res, f"{c.name} family b, passes = 2")
    if tc.conv_path(c)["row64"]:
        env = dict(c.env, VD3D_ROW64="0")
        got = run_conv(c, (x.half(), torch.zeros_like(x).half()), (whi, torch.zeros_like(whi)), osc, b, r, env=env)
        assert_exact(got, want, f"{c.name} family a, VD3D_ROW64=0")


def normal_conv_run(c, seed, wmax=None):
    """random-normal operands of row c and their planes; wmax: the weights rescaled to that largest magnitude"""
    Ho, Wo = tc.out_hw(c.H, c.W, c.KH, c.KW, c.stride, c.pad, c.dil)
    x, w, b, r = tc.normal_operands(c.B, c.Cin, c.H, c.W, c.Cout, c.KH, c.KW, res_shape(c, c.B, Ho, Wo), seed)
    if wmax is not None:
        w = w / w.abs().max() * wmax
    if r is not None:
        r = r.float().double()
    b = b.float().double()
    cin64 = tc.cdiv(c.Cin, 64) * 64
    whi, wlo, osc = E.fp16_split_scaled(tc.pack_weight(w, cin64))
    return x, w, b, r, tc.split16(x), (whi, wlo), osc


def check_normal(got, want, bound, fam, name):
    f32, hi, lo = got
    if f32 is not None:
        note_ratio(fam, name, tc.err_ratio(f32, want, bound))
        if hi is not None:
            h = f32.half()
            assert torch.equal(hi, h) and torch.equal(lo, (f32 - h.float()).half()), f"{name}: output planes are not the split of the fp32 output"
    else:
        note_ratio(fam, name + " (planes)", tc.err_ratio(hi.double() + lo.double(), want, bound + tc.planes_bound(want, bound)))


@pytest.mark.parametrize("c", tc.CONV_CASES, ids=lambda c: c.name)
def test_conv_normal_within_bound(c):
    x, w, b, r, xp, wp, osc = normal_conv_run(c, 20)
    want, mags = tc.conv_ref(x, w, b, r, c.stride, c.pad, c.dil, c.relu, c.res == "up")
    p = tc.conv_path(c)
    bound = tc.tc16_bound(mags, p["KB"], p["chunk"], osc, r, b, c.res == "up", c.res == "planes")
    got = run_conv(c, xp, wp, osc, b, r)
    check_normal(got, want, bound, "conv2d_tc16", c.name)
    # the schedules the engine claims give the same bits: the row-strip kernel against conv2d_tcp_kernel, the ring-staged accumulator against
    # the separate tile (skipped where the switch cannot move the accumulator: at BN = 32 the ring gains no stage, so it never holds the tile)
    if p["row64"]:
        assert_same_bits(got, run_conv(c, xp, wp, osc, b, r, env=dict(c.env, VD3D_ROW64="0")), f"{c.name}: VD3D_ROW64=0")
    else:
        flip = "0" if p["staging"] != "sep" else "1"
        if tc.conv_path(c, env_override={"VD3D_TC_TILE_IN_RING": flip})["staging"] != p["staging"]:
            alt = run_conv(c, xp, wp, osc, b, r, env=dict(c.env, VD3D_TC_TILE_IN_RING=flip))
            assert_same_bits(got, alt, f"{c.name}: VD3D_TC_TILE_IN_RING={flip}")


@pytest.mark.parametrize("wmax", [2.0 ** -12, 2.0 ** 39], ids=["k_clamped_at_24", "k_clamped_at_-24"])
def test_conv_weight_scale_clamp_within_bound(wmax):
    """weights so small (large) that the power-of-two weight scale is clamped at 2^24 (2^-24): max |w| 2^-12 scales to 2^12 only, and the
    planes of the smaller weights go subnormal; max |w| 2^39 scales to 2^15"""
    c = tc.CONV_CASES[[c.name for c in tc.CONV_CASES].index("bn48_1x7_kb7")]._replace(res="f32", outf="f32")
    x, w, b, r, xp, wp, osc = normal_conv_run(c, 21, wmax)
    assert osc == (2.0 ** -24 if wmax < 1 else 2.0 ** 24)
    want, mags = tc.conv_ref(x, w, b, r, c.stride, c.pad, c.dil, c.relu)
    p = tc.conv_path(c)
    check_normal(run_conv(c, xp, wp, osc, b, r), want, tc.tc16_bound(mags, p["KB"], p["chunk"], osc, r, b), "conv2d_tc16", f"max |w| {wmax:g}")


def test_every_tile_width_and_v8_are_bit_identical():
    """one conv with a ragged Cout % 8 == 4 tail and an upsampled residual: every requested tile width (16 .. 128, and 144 / 192 / 256, which
    run as halves) gives the same bits; so do the v8 stores against the scalar ones (32-byte against 16-byte aligned bias)"""
    c = tc.CONV_CASES[[c.name for c in tc.CONV_CASES].index("bn80_req144_up")]
    x, w, b, r, xp, wp, osc = normal_conv_run(c, 22)
    ref = None
    for bn in (16, 32, 48, 64, 80, 96, 112, 128, 144, 192, 256):
        got = run_conv(c._replace(bn=bn), xp, wp, osc, b, r)
        ref = ref or got
        assert_same_bits(got, ref, f"bn {bn}")
    for name, other in (("row64_cin56_v8off", "row64_cin56_v8on"), ("bn64_units180_kb1", None)):
        c = tc.CONV_CASES[[c.name for c in tc.CONV_CASES].index(name)]
        x, w, b, r, xp, wp, osc = normal_conv_run(c, 23)
        a = run_conv(c, xp, wp, osc, b, r)
        if other:
            c2 = tc.CONV_CASES[[c.name for c in tc.CONV_CASES].index(other)]
            assert tc.conv_path(c)["v8"] != tc.conv_path(c2)["v8"]
            alt = run_conv(c2, xp, wp, osc, b, r)
        else:
            assert tc.conv_path(c)["v8"] == 1 and tc.conv_path(c._replace(bias_mis=True))["v8"] == 0
            alt = run_conv(c, xp, wp, osc, b, r, bias_mis=True)
        assert_same_bits(a, alt, f"{name}: v8 on / off")


def test_residual_is_added_before_the_bias():
    """acc * out_scale + residual, then + bias: with a residual that cancels the accumulator exactly (2^17 - 64) and a bias of 2^-9, only that
    order gives the bias back (the accumulator plus the bias rounds the bias away)"""
    B, Cin, H, W, Cout = 1, 64, 3, 20, 16
    x = torch.full((B, Cin, H, W), 2047.0, dtype=torch.float64)
    w = torch.ones(Cout, Cin, 1, 1, dtype=torch.float64)
    b = torch.full((Cout,), 2.0 ** -9, dtype=torch.float64)
    acc = torch.nn.functional.conv2d(x, w)
    r = -acc
    whi, wlo, osc = E.fp16_split_scaled(tc.pack_weight(w, 64))
    for outf in ("f32", "both"):
        got = run_tc16(B, Cin, Cin, 0, [(x.half(), torch.zeros_like(x).half())], Cout, Cout + 8, 8, 1, 1, 1, 0, 1, (whi, wlo), osc, b, False,
                       [r], "f32", outf, False, 0, what="residual order")[0]
        assert_exact(got, b.view(1, -1, 1, 1).expand_as(acc).contiguous(), f"residual before bias ({outf})")


# ---- multi-level launches ------------------------------------------------------------------------------------------------------------------
def multi_setup(c, kind, seed):
    ohws = tc.multi_out_hws(c)
    levels = []
    for l, ((H, W), (Ho, Wo)) in enumerate(zip(c.hws, ohws)):
        rs = None if c.res == "none" else ((c.B, c.Cout, Ho // 2, Wo // 2) if c.res == "up" else (c.B, c.Cout, Ho, Wo))
        ops = (tc.exact_operands if kind == "exact" else tc.normal_operands)(c.B, c.Cin, H, W, c.Cout, c.KH, c.KW, rs, seed + l)
        levels.append(ops)
    w, b = levels[0][1], levels[0][2].float().double()
    xs = [lv[0] for lv in levels]
    rs = [lv[3].float().double() if lv[3] is not None else None for lv in levels]
    return xs, w, b, rs


def run_multi(c, xps, wp, osc, b, rs, what, bn=None):
    return run_tc16(c.B, c.Cin, c.in_cs, c.in_co, xps, c.Cout, c.out_cs, c.out_co, c.KH, c.KW, c.stride, c.pad, 1, wp, osc, b, False,
                    rs if c.res != "none" else None, c.res, c.outf, c.relu, c.bn if bn is None else bn, what=what)


@pytest.mark.parametrize("c", tc.MULTI_CASES, ids=lambda c: c.name)
def test_multi_level_plane_products_exact(c):
    xs, w, b, rs = multi_setup(c, "exact", 30)
    whi, wlo, osc = E.fp16_split_scaled(tc.pack_weight(w, tc.cdiv(c.Cin, 64) * 64))
    assert not bool(wlo.float().any())
    wants = [tc.conv_ref(x, w, b, r, c.stride, c.pad, 1, c.relu, c.res == "up")[0] for x, r in zip(xs, rs)]
    for fam in "abcd":
        fx = [plane_families(x.half(), whi)[fam] for x in xs]
        got = run_multi(c, [f[:2] for f in fx], fx[0][2:], osc, b, rs, f"{c.name} family {fam}")
        for l, (g, want, r) in enumerate(zip(got, wants, rs)):
            exp = tc.epilogue_ref(torch.zeros_like(want), b, r, c.relu, c.res == "up") if fam == "d" else want
            assert_exact(g, exp, f"{c.name} level {l} family {fam}")


@pytest.mark.parametrize("c", tc.MULTI_CASES, ids=lambda c: c.name)
def test_multi_level_normal_within_bound_and_equal_to_per_level_launches(c):
    xs, w, b, rs = multi_setup(c, "normal", 40)
    whi, wlo, osc = E.fp16_split_scaled(tc.pack_weight(w, tc.cdiv(c.Cin, 64) * 64))
    xps = [tc.split16(x) for x in xs]
    got = run_multi(c, xps, (whi, wlo), osc, b, rs, c.name)
    p = tc.multi_path(c)
    for l, (g, x, r) in enumerate(zip(got, xs, rs)):
        want, mags = tc.conv_ref(x, w, b, r, c.stride, c.pad, 1, c.relu, c.res == "up")
        check_normal(g, want, tc.tc16_bound(mags, p["KB"], p["chunk"], osc, r, b, c.res == "up"), "multi-level", f"{c.name} level {l}")
        one = run_tc16(c.B, c.Cin, c.in_cs, c.in_co, [xps[l]], c.Cout, c.out_cs, c.out_co, c.KH, c.KW, c.stride, c.pad, 1, (whi, wlo), osc, b,
                       False, [r] if r is not None else None, c.res, c.outf, c.relu, p["BN"], what=f"{c.name} level {l} alone")[0]
        assert_same_bits(g, one, f"{c.name} level {l}: multi-level launch against the level alone")


# ---- vd3d_convtranspose2d_tc16 ---------------------------------------------------------------------------------------------------------------
def run_convt(c, xp, wt, b, outf=None, relu=None):
    """wt: float64 [Cin, Cout, 4, 4] (packed here through engine.convtranspose_phase_matrix), or a (w_hi, w_lo, out_scale) triple"""
    outf = c.outf if outf is None else outf
    relu = c.relu if relu is None else relu
    if isinstance(wt, tuple):
        whi, wlo, osc = wt
    else:
        whi, wlo, osc = E.fp16_split_scaled(E.convtranspose_phase_matrix(wt, tc.cdiv(c.Cin, 64) * 64))
    xh, xl = slot(xp[0], c.in_cs, c.in_co, INF, torch.float16), slot(xp[1], c.in_cs, c.in_co, INF, torch.float16)
    whi, wlo = whi.cuda(), wlo.cuda()
    bbuf, bias = bias_slot(b, False)
    Ho, Wo = 2 * c.H, 2 * c.W
    out = Outputs((c.B + 1) * Ho * Wo, c.out_cs, outf in ("f32", "both"), outf in ("planes", "both"))
    call("vd3d_convtranspose2d_tc16", xh.data_ptr(), xl.data_ptr(), c.B, c.H, c.W, c.Cin, c.in_cs, c.in_co, whi.data_ptr(), wlo.data_ptr(),
         osc, bias.data_ptr(), out.f32.data_ptr() if out.f32 is not None else None, out.hi.data_ptr() if out.hi is not None else None,
         out.lo.data_ptr() if out.lo is not None else None, c.Cout, c.out_cs, c.out_co, 1 if relu else 0, c.bn, None)
    torch.cuda.synchronize()
    out.check_untouched([(0, c.B * Ho * Wo)], c.out_co, c.Cout, c.name)
    return out.get(0, c.B, Ho, Wo, c.out_co, c.Cout)


@pytest.mark.parametrize("c", tc.CONVT_CASES, ids=lambda c: c.name)
def test_convtranspose_plane_products_exact(c):
    x, wt, b, _ = tc.exact_operands(c.B, c.Cin, c.H, c.W, c.Cout, 4, 4, None, 50, w_layout="convt")
    want, _ = tc.convt_ref(x, wt, b, c.relu)
    whi, wlo, osc = E.fp16_split_scaled(E.convtranspose_phase_matrix(wt, tc.cdiv(c.Cin, 64) * 64))
    assert osc == 2.0 ** -14 and not bool(wlo.float().any())
    for fam, (xh, xl, wh, wl) in plane_families(x.half(), whi).items():
        got = run_convt(c, (xh, xl), (wh, wl, osc), b)
        exp = tc.epilogue_ref(torch.zeros_like(want), b, None, c.relu) if fam == "d" else want
        assert_exact(got, exp, f"{c.name} family {fam}")


@pytest.mark.parametrize("c", tc.CONVT_CASES, ids=lambda c: c.name)
def test_convtranspose_normal_within_bound(c):
    x, wt, b, _ = tc.normal_operands(c.B, c.Cin, c.H, c.W, c.Cout, 4, 4, None, 60, w_layout="convt")
    b = b.float().double()
    want, mags = tc.convt_ref(x, wt, b, c.relu)
    p = tc.convt_path(c)
    osc = E.fp16_split_scaled(E.convtranspose_phase_matrix(wt, p["cin_pad"]))[2]
    got = run_convt(c, tc.split16(x), wt, b)
    check_normal(got, want, tc.tc16_bound(mags, p["KB"], p["chunk"], osc, None, b), "convtranspose2d_tc16", c.name)


# ---- 3xTF32 (vd3d_conv2d_tc) -----------------------------------------------------------------------------------------------------------------
def trunc13(t):
    return (t.float().contiguous().view(torch.int32) & -8192).view(torch.float32)


def run_tf32(c, x_hi, x_lo, w, b, r):
    Ho, Wo = tc.out_hw(c.H, c.W, c.K, c.K, 1, c.pad, c.dil)
    xb = slot(x_hi, c.in_cs, c.in_co, INF, torch.float32)
    xl = slot(x_lo, c.in_cs, c.in_co, INF, torch.float32)
    wk = tc.pack_weight(w, c.Cin).float()
    whi, wlo = (t.cuda() for t in E.tf32_split(wk))
    bbuf, bias = bias_slot(b, False)
    rb = slot(r, c.out_cs, c.out_co, INF, torch.float32) if r is not None else None
    npix = (c.B + 1) * Ho * Wo
    out = Outputs(npix, c.out_cs, True, False)
    olo = torch.full((npix, c.out_cs), SENT32, device="cuda") if c.out_lo else None
    call("vd3d_conv2d_tc", xb.data_ptr(), xl.data_ptr() if c.passes == 3 else None, c.B, c.H, c.W, c.Cin, c.in_cs, c.in_co,
         whi.data_ptr(), wlo.data_ptr(), bias.data_ptr(), c.K, c.K, c.pad, c.dil,
         rb.data_ptr() if rb is not None else None, c.out_cs if rb is not None else 0, c.out_co if rb is not None else 0,
         out.f32.data_ptr(), olo.data_ptr() if olo is not None else None, c.Cout, c.out_cs, c.out_co, 1 if c.relu else 0, c.passes, c.bn, None)
    torch.cuda.synchronize()
    out.check_untouched([(0, c.B * Ho * Wo)], c.out_co, c.Cout, c.name)
    got = out.get(0, c.B, Ho, Wo, c.out_co, c.Cout)[0]
    if olo is not None:
        m = torch.ones(olo.shape, dtype=torch.bool, device="cuda")
        m[:c.B * Ho * Wo, c.out_co:c.out_co + c.Cout] = False
        assert bool((olo[m] == SENT32).all()), f"{c.name}: the lo companion was written outside its slice"
        lo = nchw(olo[:c.B * Ho * Wo, c.out_co:c.out_co + c.Cout].reshape(c.B, Ho, Wo, c.Cout)).cpu()
        assert torch.equal(lo, got - trunc13(got)), f"{c.name}: the tf32 lo companion is not value - trunc13(value)"
    return got


@pytest.mark.parametrize("c", tc.TF32_CASES, ids=lambda c: c.name)
def test_tf32_exact_and_within_bound(c):
    Ho, Wo = tc.out_hw(c.H, c.W, c.K, c.K, 1, c.pad, c.dil)
    rs = (c.B, c.Cout, Ho, Wo) if c.res else None
    x, w, b, r = tc.exact_operands(c.B, c.Cin, c.H, c.W, c.Cout, c.K, c.K, rs, 70)
    want, _ = tc.conv_ref(x, w, b, r, 1, c.pad, c.dil, c.relu)
    z = torch.zeros_like(x)
    assert_exact((run_tf32(c, x, z, w, b, r), None, None), want, f"{c.name} exact")
    # x in the lo companion only: the A_lo * W_hi product (passes 3); one pass does not read it
    lo_only = want if c.passes == 3 else tc.epilogue_ref(torch.zeros_like(want), b, r, c.relu)
    assert_exact((run_tf32(c, z, x, w, b, r), None, None), lo_only, f"{c.name} x in lo only")
    x, w, b, r = tc.normal_operands(c.B, c.Cin, c.H, c.W, c.Cout, c.K, c.K, rs, 71)
    x, w, b = x.float().double(), w.float().double(), b.float().double()
    r = r.float().double() if r is not None else None
    want, mags = tc.conv_ref(x, w, b, r, 1, c.pad, c.dil, c.relu)
    p = tc.tf32_path(c)
    got = run_tf32(c, x, x - trunc13(x).double(), w, b, r)
    note_ratio(f"conv2d_tc passes={c.passes}", c.name, tc.err_ratio(got, want, tc.tf32_bound(mags, p["KB"], p["chunk"], c.passes, r, b)))


# ---- the fp16 range flag at tile edges -------------------------------------------------------------------------------------------------------
def impulse_conv(B, Cin, H, W, Cout, KH, KW, stride, pad, dil, target, xv, wv):
    """x zero but one input pixel (channel 0), w zero but one tap of output channel co: output (b, co, ho, wo) = xv * wv, all others 0"""
    b_, co, ho, wo = target
    x = torch.zeros(B, Cin, H, W, dtype=torch.float64)
    w = torch.zeros(Cout, Cin, KH, KW, dtype=torch.float64)
    for kh in range(KH):
        for kw in range(KW):
            hi, wi = ho * stride - pad + kh * dil, wo * stride - pad + kw * dil
            if 0 <= hi < H and 0 <= wi < W:
                x[b_, 0, hi, wi] = xv
                w[co, 0, kh, kw] = wv
                return x, w
    raise AssertionError("no in-image tap")


# (name, Cin, H, W, Cout, KH, stride, pad, bn, target (b, co, ho, wo)): the value lands in ...
RANGE_CASES = [
    ("ragged_n_tile_last_column", 64, 12, 20, 136, 3, 1, 1, 144, (0, 135, 5, 7)),     # BN 80: 56 of the second tile's 80 columns are valid
    ("cout8_tail", 64, 12, 20, 132, 3, 1, 1, 144, (0, 129, 3, 3)),                    # channels 128..131: the Cout % 8 == 4 group
    ("ragged_m_tile_last_pixel", 40, 25, 41, 48, 3, 2, 1, 0, (1, 47, 12, 20)),        # Ho 13 x Wo 21: last pixel of the last M tile
]
RANGE_VALUES = [((4095.0, 16.0), True), ((-4095.0, 16.0), True), ((65519.0, 1.0), False)]      # 65520, -65520 and 65519


@pytest.mark.parametrize("rc", RANGE_CASES, ids=lambda rc: rc[0])
def test_fp16_range_flag_at_tile_edges(rc):
    name, Cin, H, W, Cout, K, s, pad, bn, target = rc
    B = target[0] + 1
    c = tc.Conv(name, B, Cin, Cin, 0, H, W, Cout, Cout + 4, 0, K, K, s, pad, 1, bn, "none", "both", False, False, (), "")
    b = torch.zeros(Cout, dtype=torch.float64)
    for (xv, wv), flagged in RANGE_VALUES:
        x, w = impulse_conv(B, Cin, H, W, Cout, K, K, s, pad, 1, target, xv, wv)
        whi, wlo, osc = E.fp16_split_scaled(tc.pack_weight(w, tc.cdiv(Cin, 64) * 64))
        for outf, expect in (("both", flagged), ("f32", False)):
            flag_clear()
            got = run_conv(c._replace(outf=outf), tc.split16(x), (whi, wlo), osc, b, None)
            assert float(got[0][target]) == xv * wv and float(got[0].abs().sum()) == abs(xv * wv), name
            assert E.fp16_range_overflowed() == expect, (name, xv * wv, outf)


def test_fp16_range_flag_in_one_level_and_one_phase():
    # level 1 of a three-level launch
    c = tc.MULTI_CASES[1]._replace(outf="both", res="none")
    ohws = tc.multi_out_hws(c)
    b = torch.zeros(c.Cout, dtype=torch.float64)
    for (xv, wv), flagged in RANGE_VALUES:
        xs = [torch.zeros(c.B, c.Cin, H, W, dtype=torch.float64) for H, W in c.hws]
        x1, w = impulse_conv(c.B, c.Cin, *c.hws[1], c.Cout, c.KH, c.KW, c.stride, c.pad, 1, (0, c.Cout - 1, ohws[1][0] - 1, 0), xv, wv)
        xs[1] = x1
        whi, wlo, osc = E.fp16_split_scaled(tc.pack_weight(w, 64))
        for outf, expect in (("both", flagged), ("f32", False)):
            flag_clear()
            got = run_multi(c._replace(outf=outf), [tc.split16(x) for x in xs], (whi, wlo), osc, b, None, "range flag level 1")
            assert float(got[1][0].abs().max()) == abs(xv * wv) and float(got[0][0].abs().max()) == 0.0
            assert E.fp16_range_overflowed() == expect, ("level 1", xv * wv, outf)
    # phase (1, 0) of a transposed conv: tap (a, c) = (0, 1) is Wt[:, :, 2, 1]; input pixel (H - 1, W - 1) -> output (2 H - 1, 2 W - 2)
    c = tc.CONVT_CASES[1]
    b = torch.zeros(c.Cout, dtype=torch.float64)
    for (xv, wv), flagged in RANGE_VALUES:
        x = torch.zeros(c.B, c.Cin, c.H, c.W, dtype=torch.float64)
        x[c.B - 1, 0, c.H - 1, c.W - 1] = xv
        wt = torch.zeros(c.Cin, c.Cout, 4, 4, dtype=torch.float64)
        wt[0, 5, 2, 1] = wv
        for outf, expect in (("both", flagged), ("f32", False)):
            flag_clear()
            v = run_convt(c, tc.split16(x), wt, b, outf=outf)[0]
            assert float(v[c.B - 1, 5, 2 * c.H - 1, 2 * c.W - 2]) == xv * wv and float(v.abs().sum()) == abs(xv * wv)
            assert E.fp16_range_overflowed() == expect, ("phase (1, 0)", xv * wv, outf)
