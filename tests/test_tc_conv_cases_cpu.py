"""The case tables, references and bounds of tests/tc_conv_cases.py, checked without a GPU:
  * every row reaches the path its name and `reach` string state (tile width, staging, v8, row-strip kernel, L2 blocking), and the restated
    tile pickers equal the library's exported ones;
  * the tables reach every tile instantiation, requested width, tail, stride, dilation, kernel shape, channel offset, k-block count,
    residual and output form and switch setting the engine has;
  * the exact operand families are exact: every partial sum on one dyadic grid below 2^20 grid units, weights that fp16_split_scaled keeps
    whole in the hi plane;
  * the comparisons fail on known-wrong arithmetic: an output pixel read one tap off, the A_lo * W_hi product dropped (passes = 2), the
    residual added after the bias."""
import math

import pytest
import torch
import torch.nn.functional as F

import tc_conv_cases as tc
from visualdet3d_b200 import engine as E

ALL_SINGLE = [(c, tc.conv_path(c)) for c in tc.CONV_CASES]


@pytest.mark.parametrize("c", tc.CONV_CASES, ids=lambda c: c.name)
def test_conv_row_reaches_its_path(c):
    assert tc.path_name(tc.conv_path(c)) == c.reach
    Ho, Wo = tc.out_hw(c.H, c.W, c.KH, c.KW, c.stride, c.pad, c.dil)
    assert Ho > 0 and Wo > 0 and c.in_cs >= c.in_co + c.Cin and c.out_cs >= c.out_co + c.Cout
    assert c.Cin % 8 == 0 and c.in_cs % 8 == 0 and c.in_co % 8 == 0 and c.out_cs % 4 == 0 and c.out_co % 4 == 0 and c.Cout % 4 == 0
    if c.res == "up":
        assert Ho % 2 == 0 and Wo % 2 == 0


@pytest.mark.parametrize("c", tc.MULTI_CASES, ids=lambda c: c.name)
def test_multi_level_row_reaches_its_path(c):
    assert tc.path_name(tc.multi_path(c)) == c.reach
    assert 2 <= len(c.hws) <= tc.TC_MAX_LEVELS
    if c.res == "up":
        assert all(h % 2 == 0 and w % 2 == 0 for h, w in tc.multi_out_hws(c))


@pytest.mark.parametrize("c", tc.CONVT_CASES, ids=lambda c: c.name)
def test_convtranspose_row_reaches_its_path(c):
    assert tc.path_name(tc.convt_path(c)) == c.reach and c.Cout % 16 == 0


@pytest.mark.parametrize("c", tc.TF32_CASES, ids=lambda c: c.name)
def test_tf32_row_reaches_its_path(c):
    assert tc.path_name(tc.tf32_path(c)) == c.reach and c.Cin % 32 == 0


def test_restated_pickers_equal_the_library():
    from visualdet3d_b200 import _lib
    lib = _lib.load()
    for cout in list(range(4, 1500, 4)) + [2048, 4096]:
        assert lib.vd3d_tc_pick_bn(cout) == tc.pick_bn_tf32(cout), cout
        assert lib.vd3d_tc_pick_bn_persistent(cout) == tc.pick_bn_persistent(cout), cout
    assert [tc.fit_bn(b) for b in (16, 128, 144, 192, 256)] == [16, 128, 80, 96, 128]
    # the cost picker: a single tile up to 128 columns, then the cheapest rounds x (BN + 64)
    assert tc.pick_bn_cost(100, 1) == 112 and tc.pick_bn_cost(144, 4) == 64 and tc.pick_bn_cost(256, 200) == 128


def test_ring_layouts_are_the_documented_ones():
    """stages with the accumulator staged in the ring against a separate tile (DESIGN 3.1: 128 columns 2 -> 3, 112: 2 -> 3, 96 / 80 / 64:
    3 -> 4), and split staging only at 112 and 128 columns"""
    for bn, sep, ring, split in ((128, 2, 3, True), (112, 2, 3, True), (96, 3, 4, False), (80, 3, 4, False), (64, 3, 4, False),
                                 (48, 4, 5, False), (32, 5, 5, False), (16, 5, 6, False)):
        assert tc.ring_layout(bn, "0")[:2] == (sep, False)
        st, in_ring, sp = tc.ring_layout(bn)
        assert (st, in_ring or st == sep, sp) == (ring, True, split), bn


def test_tables_cover_every_path_and_edge():
    cs = tc.CONV_CASES
    paths = [p for _, p in ALL_SINGLE]
    # every tile instantiation, on conv2d_tcp_kernel and (up to 64 columns) on the row-strip kernel; requested widths that run as halves
    assert {p["BN"] for p in paths if not p["row64"]} == {16, 32, 48, 64, 80, 96, 112, 128}
    assert {p["BN"] for p in paths if p["row64"]} == {16, 32, 48, 64}
    assert {144, 192, 256} <= {c.bn for c in cs}
    assert {p["staging"] for p in paths if not p["row64"]} == {"sep", "ring", "split"}
    assert any(p["mblock"] for p in paths) and any(p["n_tiles"] * p["m_tiles"] > tc.NUM_SMS for p in paths)
    # Cout tails and the v8 / scalar stores on one conv
    assert {c.Cout % 16 for c in cs} == {0, 4, 8, 12} and any(c.Cout % 8 == 4 for c in cs)
    assert {c.out_co % 8 for c in cs} == {0, 4} and {p["v8"] for p in paths} == {0, 1}
    assert any(c.bias_mis and c.out_co % 8 == 0 and c.out_cs % 8 == 0 for c in cs)
    pairs = {}
    for c, p in ALL_SINGLE:
        pairs.setdefault((c.B, c.Cin, c.H, c.W, c.Cout, c.KH, c.KW, c.stride, c.pad, c.dil), set()).add(p["v8"])
    assert any(v == {0, 1} for v in pairs.values())
    # M edges
    dims = [(c.B * h * w, h, w) for c in cs for h, w in [tc.out_hw(c.H, c.W, c.KH, c.KW, c.stride, c.pad, c.dil)]]
    assert 1 in {m for m, _, _ in dims} and {1, 127} <= {m % 128 for m, _, _ in dims}
    assert any(h < tc.TC_TH or w < tc.TC_TW for _, h, w in dims)
    # geometry
    assert {1, 2, 3, 4} == {c.stride for c in cs}
    assert any(c.pad == 0 for c in cs) and any(c.pad > max(c.KH, c.KW) // 2 for c in cs)
    assert {(d, s) for c in cs for d, s in [(c.dil, c.stride)] if d > 1} >= {(2, 1), (2, 2), (3, 1), (3, 2)}
    assert {(1, 1), (3, 3), (5, 5), (1, 3), (3, 1), (7, 1), (1, 7)} <= {(c.KH, c.KW) for c in cs}
    assert {8, 16, 40, 56, 64, 72, 136} <= {c.Cin for c in cs} and {0, 8, 24} <= {c.in_co for c in cs}
    assert {c.Cin % 64 for c in cs if c.in_co > 0} >= {8, 16, 40, 56}
    # k-block counts against the promotion chunk
    kb = [(p["KB"], p["chunk"]) for p in paths]
    assert any(k == 1 for k, _ in kb) and any(k < ch for k, ch in kb if k > 1) and any(ch > k for k, ch in kb if ch == 64)
    assert {k % ch for k, ch in kb if ch == 4} >= {1, 3} and {ch for _, ch in kb} == {1, 4, 64}
    # epilogue forms and switches
    assert {c.res for c in cs} == {"none", "f32", "planes", "up"} and {c.outf for c in cs} == {"f32", "planes", "both"}
    assert {c.relu for c in cs} == {True, False}
    assert {dict(c.env).get("VD3D_TC_TILE_IN_RING") for c in cs} >= {"0", "1"}
    # multi-level: 2 .. 5 levels, a 1x1 level, ragged levels, an upsampled residual, planes output, more units than SMs
    ms = tc.MULTI_CASES
    assert {len(c.hws) for c in ms} == {2, 3, 4, 5} and any((1, 1) in tc.multi_out_hws(c) for c in ms)
    assert any(h % tc.TC_TH or w % tc.TC_TW for c in ms for h, w in tc.multi_out_hws(c))
    assert {c.res for c in ms} >= {"up", "f32"} and any(c.outf != "f32" for c in ms)
    assert any(tc.multi_path(c)["m_tiles"] * tc.multi_path(c)["n_tiles"] > tc.NUM_SMS for c in ms)
    # transposed conv: H or W = 1, odd sizes, Cin % 64, Cout off 128 through the picker, planes-only, ReLU off, a channel slice
    ts = tc.CONVT_CASES
    assert any(c.H == 1 or c.W == 1 for c in ts) and any(c.H % 2 and c.W % 2 for c in ts) and any(c.Cin % 64 for c in ts)
    assert any(c.bn == 0 and c.Cout % 128 and c.Cout > 128 for c in ts)
    assert any(c.outf == "planes" for c in ts) and any(not c.relu for c in ts) and any(c.out_co > 0 for c in ts)
    # 3xTF32: passes 1 and 3, the lo companion, several tile widths
    assert {c.passes for c in tc.TF32_CASES} == {1, 3} and any(c.out_lo for c in tc.TF32_CASES)
    assert len({tc.tf32_path(c)["BN"] for c in tc.TF32_CASES}) >= 4


def test_row64_rows_also_run_on_the_persistent_kernel():
    for c, p in ALL_SINGLE:
        if p["row64"]:
            q = tc.conv_path(c, env_override={"VD3D_ROW64": "0"})
            assert not q["row64"] and q["BN"] == p["BN"]
    assert sum(p["row64"] for _, p in ALL_SINGLE) >= 4
    # a 3x3 / stride-1 / pad-1 64-channel conv is taken off the row-strip kernel by a second N tile, passes = 2, or an upsampled residual
    c = tc.CONV_CASES[0]
    assert not tc.conv_path(c._replace(bn=16, Cout=20))["row64"] and not tc.conv_path(c, passes=2)["row64"]
    assert not tc.conv_path(c._replace(res="up"))["row64"]


# ---- exact operands ----------------------------------------------------------------------------------------------------------------------
def _exact_rows():
    for c in tc.CONV_CASES:
        yield c.name, c.Cin, c.Cout, c.KH, c.KW
    for c in tc.MULTI_CASES:
        yield c.name, c.Cin, c.Cout, c.KH, c.KW
    for c in tc.CONVT_CASES:
        yield c.name, c.Cin, c.Cout, 2, 2


@pytest.mark.parametrize("row", list(_exact_rows()), ids=lambda r: r[0])
def test_exact_families_are_exact(row):
    name, Cin, Cout, KH, KW = row
    x, w, b, r = tc.exact_operands(1, Cin, 8, 9, Cout, KH, KW, (1, Cout, 9 - KH, 10 - KW), 10)
    # every product is a multiple of 1/8 (2^11 after the weight scale 2^14), every partial sum stays below 2^20 grid units
    assert torch.equal(x, x.round()) and torch.equal(w * 8, (w * 8).round()) and float(w.abs().max()) == 1.0
    assert torch.equal(b * 8, (b * 8).round()) and torch.equal(r, r.round())
    assert tc.exact_grid_limit(KH * KW * Cin) < 2 ** 20
    # fp16: x whole and exact; the weights survive the scaled split whole in the hi plane, lo = 0
    assert torch.equal(x.half().double(), x)
    cin64 = tc.cdiv(Cin, 64) * 64
    hi, lo, osc = E.fp16_split_scaled(tc.pack_weight(w, cin64))
    assert osc == 2.0 ** -14 and not bool(lo.float().any())
    assert torch.equal(hi.double() * osc, tc.pack_weight(w, cin64))
    # a float32 conv of the exact operands (any summation order) equals float64
    want, _ = tc.conv_ref(x, w, b, r, 1, 0, 1, False)
    got = F.conv2d(x.float(), w.float(), None) + r.float() + b.float().view(1, -1, 1, 1)
    assert torch.equal(got.double(), want)


def test_transposed_reference_equals_the_phase_packing():
    """the float64 transposed-conv reference (F.conv_transpose2d) and the engine's phase matrix describe the same operator"""
    x, wt, b, _ = tc.exact_operands(2, 40, 3, 5, 16, 4, 4, None, 3, w_layout="convt")
    want, _ = tc.convt_ref(x, wt, b, False)
    m = E.convtranspose_phase_matrix(wt, 64).reshape(4, 16, 4, 64)
    got = torch.zeros_like(want)
    for r in (0, 1):
        for s in (0, 1):
            wp = m[2 * r + s].reshape(16, 2, 2, 64)[..., :40].permute(0, 3, 1, 2)
            xp = F.pad(x, (1 - s, s, 1 - r, r))
            got[:, :, r::2, s::2] = F.conv2d(xp, wp)
    assert torch.equal(got + b.view(1, -1, 1, 1), want)


# ---- the comparisons catch known-wrong arithmetic ---------------------------------------------------------------------------------------------
def _normal_case(c, seed=5, wmax=None):
    Ho, Wo = tc.out_hw(c.H, c.W, c.KH, c.KW, c.stride, c.pad, c.dil)
    x, w, b, r = tc.normal_operands(c.B, c.Cin, c.H, c.W, c.Cout, c.KH, c.KW, (c.B, c.Cout, Ho, Wo), seed)
    if wmax is not None:
        w = w / w.abs().max() * wmax
    b, r = b.float().double(), r.float().double()
    cin64 = tc.cdiv(c.Cin, 64) * 64
    whi, wlo, osc = E.fp16_split_scaled(tc.pack_weight(w, cin64))
    unpack = lambda t: t.double().reshape(c.Cout, c.KH, c.KW, cin64)[..., :c.Cin].permute(0, 3, 1, 2)
    xh, xl = tc.split16(x)
    p = tc.conv_path(c)
    want, mags = tc.conv_ref(x, w, b, r, c.stride, c.pad, c.dil, c.relu)
    bound = tc.tc16_bound(mags, p["KB"], p["chunk"], osc, r, b)
    planes = (xh.double(), xl.double(), unpack(whi), unpack(wlo), osc)
    return x, w, b, r, planes, want, bound


CPU_ROWS = ["bn48_1x7_kb7", "bn32_m255_d2_chunk1", "bn112_s4_pad2"]


@pytest.mark.parametrize("name", CPU_ROWS)
def test_bound_holds_for_the_engine_arithmetic_restated(name):
    """the three products in float64, rounded to float32 once, plus the float32 epilogue: inside the bound (the epilogue's two roundings
    alone reach half of it where every tap is padding)"""
    c = tc.CONV_CASES[[c.name for c in tc.CONV_CASES].index(name)]
    x, w, b, r, (xh, xl, wh, wl, osc), want, bound = _normal_case(c)
    acc = tc.plane_conv(xh, xl, wh, wl, osc, c.stride, c.pad, c.dil)
    got = tc.epilogue_f32(acc, b, r, c.relu)
    assert tc.err_ratio(got, want, bound) <= 1.0


@pytest.mark.parametrize("wmax, ratio", [(2.0 ** -12, 0.607), (2.0 ** 39, 0.498)])
def test_clamped_weight_rows_meet_the_bound_through_the_epilogue(wmax, ratio):
    """the GPU test's clamped-weight rows (same operands): the restated arithmetic reaches the ratio the device reports (0.607 and 0.498 on
    an H100), at an element where the accumulator is small next to residual and bias, so the error is the epilogue's two roundings,
    (acc + r) and then + b, each up to half an ulp of its result, against a bound of 2^-24 (|acc| + |r| + |b|) for each"""
    c = tc.CONV_CASES[[c.name for c in tc.CONV_CASES].index("bn48_1x7_kb7")]._replace(res="f32", outf="f32")
    x, w, b, r, (xh, xl, wh, wl, osc), want, bound = _normal_case(c, 21, wmax)
    acc = tc.plane_conv(xh, xl, wh, wl, osc, c.stride, c.pad, c.dil)
    got = tc.epilogue_f32(acc, b, r, c.relu)
    assert tc.err_ratio(got, want, bound) == pytest.approx(ratio, abs=5e-4)
    i = int(((got.double() - want).abs() / bound).argmax())
    assert abs(float(acc.reshape(-1)[i])) < 1e-3 * abs(float(r.reshape(-1)[i]))


@pytest.mark.parametrize("name", CPU_ROWS)
def test_bound_fails_when_a_pixel_reads_one_tap_off(name):
    c = tc.CONV_CASES[[c.name for c in tc.CONV_CASES].index(name)]
    x, w, b, r, (xh, xl, wh, wl, osc), want, bound = _normal_case(c)
    acc = tc.plane_conv(xh, xl, wh, wl, osc, c.stride, c.pad, c.dil)
    shifted = tc.plane_conv(torch.roll(xh, 1, 3), torch.roll(xl, 1, 3), wh, wl, osc, c.stride, c.pad, c.dil)
    h, w_ = acc.shape[2] // 2, acc.shape[3] // 2
    acc[0, :, h, w_] = shifted[0, :, h, w_]                      # one output pixel, every channel, reads the input one column off
    assert tc.err_ratio(tc.epilogue_f32(acc, b, r, c.relu), want, bound) > 1e3


@pytest.mark.parametrize("name", CPU_ROWS)
def test_bound_fails_without_the_a_lo_w_hi_product(name):
    """passes = 2 restated: A_hi W_lo + A_hi W_hi only; the activations then carry 11 significant bits"""
    c = tc.CONV_CASES[[c.name for c in tc.CONV_CASES].index(name)]
    x, w, b, r, (xh, xl, wh, wl, osc), want, bound = _normal_case(c)
    acc = tc.plane_conv(xh, xl, wh, wl, osc, c.stride, c.pad, c.dil, products=("hi_lo", "hi_hi"))
    assert tc.err_ratio(tc.epilogue_f32(acc, b, r, c.relu), want, bound) > 10
    # the exact family (b) sees it as an output of exactly bias + residual
    xe, we, be, re = tc.exact_operands(1, c.Cin, c.H, c.W, c.Cout, c.KH, c.KW, None, 1)
    z = torch.zeros_like(xe)
    acc = tc.plane_conv(z, xe, we * 2 ** 14, we * 0, 2.0 ** -14, c.stride, c.pad, c.dil, products=("hi_lo", "hi_hi"))
    want, _ = tc.conv_ref(xe, we, be, None, c.stride, c.pad, c.dil, False)
    assert not torch.equal(tc.epilogue_f32(acc, be, None, False).double(), want)


def test_exact_check_fails_when_the_residual_is_added_after_the_bias():
    """the GPU test's constructed operands: accumulator 2^17 - 64, residual its negative, bias 2^-9"""
    acc = torch.full((1, 16, 3, 20), 64 * 2047.0, dtype=torch.float64)
    b = torch.full((16,), 2.0 ** -9, dtype=torch.float64)
    want = tc.epilogue_ref(acc, b, -acc, False)
    assert torch.equal(tc.epilogue_f32(acc, b, -acc, False).double(), want)
    assert not torch.equal(tc.epilogue_f32(acc, b, -acc, False, residual_first=False).double(), want)


def test_bound_terms():
    """the accumulation term grows with the MMAs per promotion chunk and the number of chunks, as the model states"""
    assert tc.accumulation_factor(9, 4) == pytest.approx((2.0 ** -23 * 48 + 2.0 ** -24 * 3) * (1 + 2.0 ** -9))
    assert tc.accumulation_factor(1, 4) == pytest.approx((2.0 ** -23 * 12 + 2.0 ** -24) * (1 + 2.0 ** -9))
    assert tc.accumulation_factor(27, 64) > tc.accumulation_factor(27, 4) > tc.accumulation_factor(27, 1)
    assert tc.accumulation_factor(9, 4, f16=False, passes=1) < tc.accumulation_factor(9, 4, f16=False, passes=3)
    assert math.isclose(tc.SPLIT_TF32[3], 3 * 2.0 ** -20 + 2.0 ** -24)
