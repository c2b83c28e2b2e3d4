"""The case tables and float64 references of tests/support_ops_cases.py, checked without a GPU:
  * every SIMT conv row lands on the (BN, VEC) instantiation its comment names, and the table reaches every instantiation and every edge the
    kernel has (column thresholds +-4, M and K tails, strides, dilations, paddings, non-square kernels, tiny inputs, epilogue options);
  * the exact operands keep every partial sum exact in float32 (a float32 CPU conv equals the float64 reference);
  * the layout, pool, depthwise, LookGround and splitter rows reach what their comments say;
  * LookGround's restated grid is bit for bit the one torch_port.look_ground hands to grid_sample, the float64 bilinear restatement equals
    grid_sample, and the error bound is tight enough that a one-pixel shift or swapped corner weights break it."""
import math

import pytest
import torch
import torch.nn.functional as F

import support_ops_cases as sc


@pytest.mark.parametrize("c", sc.CONV_CASES, ids=lambda c: c.name)
def test_conv_row_reaches_its_instantiation(c):
    assert sc.simt_select(c.Cin, c.in_cs, c.in_co, c.Cout) == c.reach
    assert c.in_cs >= c.in_co + c.Cin and c.Cout % 4 == 0
    Ho, Wo, M, K = sc.conv_dims(c)
    assert Ho > 0 and Wo > 0


def test_conv_table_covers_every_instantiation_and_edge():
    cases = sc.CONV_CASES
    dims = [sc.conv_dims(c) for c in cases]
    assert {c.reach for c in cases} == {(bn, v) for bn in (16, 32, 64, 128) for v in (1, 4)}
    assert {4, 16, 20, 32, 36, 64, 68, 128, 132, 260} <= {c.Cout for c in cases}
    assert {1, 127} <= {m % sc.CBM for _, _, m, _ in dims} and 1 in {m for _, _, m, _ in dims}
    assert {4, 12} <= {k % sc.CBK for _, _, _, k in dims} and 3 in {k for _, _, _, k in dims}
    assert {2, 3} <= {c.stride for c in cases} and {2, 3} <= {c.dil for c in cases}
    assert 0 in {c.pad for c in cases} and any(c.pad > max(c.KH, c.KW) // 2 for c in cases)
    assert {(1, 7), (7, 1), (3, 1)} <= {(c.KH, c.KW) for c in cases}
    # an input smaller than the kernel's footprint: every output pixel reads padding
    assert any(c.H < c.dil * (c.KH - 1) + 1 and c.W < c.dil * (c.KW - 1) + 1 for c in cases)
    assert any(not c.bias for c in cases) and any(c.res for c in cases) and any(c.relu for c in cases) and any(not c.relu for c in cases)
    # the scalar gather at a non-zero channel offset
    assert any(c.reach[1] == 1 and c.in_co > 0 for c in cases)


@pytest.mark.parametrize("p", sc.PAIR_CASES, ids=lambda p: p[0])
def test_pair_rows_take_both_gathers(p):
    name, B, Cin, H, W, Cout, KH, KW, s, pad, d, in_cs = p
    bn = sc.simt_select(Cin, in_cs, 0, Cout)[0]
    assert [sc.simt_select(Cin, in_cs, co, Cout) for co in sc.PAIR_IN_CO] == [(bn, 4), (bn, 1)]
    assert in_cs >= max(sc.PAIR_IN_CO) + Cin
    assert sc.simt_select(Cin, in_cs, 4, Cout, aligned=False) == (bn, 1)
    assert {sc.simt_select(q[2], q[11], 0, q[5])[0] for q in sc.PAIR_CASES} == {16, 32, 64, 128}


@pytest.mark.parametrize("c", sc.CONV_CASES, ids=lambda c: c.name)
def test_exact_operands_are_exact_in_float32(c):
    assert sc.exact_sum_limit(c) < 2 ** 21
    x, w, b, r = sc.conv_operands(c, "exact", 0)
    want, _ = sc.conv_ref(x, w, b, r, c.stride, c.pad, c.dil, c.relu)
    got = F.conv2d(x, w, b, stride=c.stride, padding=c.pad, dilation=c.dil)
    if r is not None:
        got = got + r
    if c.relu:
        got = F.relu(got)
    assert torch.equal(got.double(), want)


def test_conv_weight_packing():
    c = sc.CONV_CASES[5]
    x, w, b, r = sc.conv_operands(c, "normal", 1)
    wk = sc.pack_conv_weight(w)
    Cin = c.Cin
    for k in (0, 1, Cin, wk.shape[0] - 1):
        tap, ci = divmod(k, Cin)
        kh, kw = divmod(tap, c.KW)
        assert torch.equal(wk[k], w[:, ci, kh, kw])


def test_conv_bound_separates_a_one_tap_slip():
    """Skipping the last K chunk or shifting a tap moves the output by far more than gamma(K + 2) S."""
    c = sc.CONV_CASES[6]
    x, w, b, r = sc.conv_operands(c, "normal", 0)
    want, S = sc.conv_ref(x, w, b, r, c.stride, c.pad, c.dil, False)
    bound = sc.gamma(sc.conv_dims(c)[3] + 2) * S
    w2 = w.clone()
    w2[:, -1, -1, -1] = 0                              # drop the last k
    slip, _ = sc.conv_ref(x, w2, b, r, c.stride, c.pad, c.dil, False)
    assert sc.err_ratio(slip, want, bound) > 1e3


@pytest.mark.parametrize("C", sc.LAYOUT_C)
def test_layout_rows(C):
    assert sc.nchw_to_nhwc_kernel(C) == ("small" if C in (1, 3, 4) else "tiled")
    hws = [h * w for h, w in sc.LAYOUT_HW]
    assert min(hws) < 32 and any(n % 32 for n in hws) and sc.LAYOUT_CO > 0


def test_layout_table_reaches_both_kernels():
    assert {sc.nchw_to_nhwc_kernel(C) for C in sc.LAYOUT_C} == {"small", "tiled"}
    assert any(C % 32 for C in sc.LAYOUT_C if C > 32)      # a ragged channel tile


def test_pool_rows():
    hs = {h for h, _ in sc.MAXPOOL3_HW} | {w for _, w in sc.MAXPOOL3_HW}
    assert {1, 2, 3} <= hs and any(v % 2 for v in hs if v > 3) and any(v % 2 == 0 for v in hs if v > 3)
    assert any(h % 2 and w % 2 for h, w in sc.MAXPOOL2_HW) and any(h % 2 != w % 2 for h, w in sc.MAXPOOL2_HW)   # floor in both / one axis
    assert all(h % 2 == 0 and w % 2 == 0 for h, w in sc.AVGPOOL_HW)
    # all-negative inputs: the -inf padding keeps every output negative, a zero-padded window would not
    x = sc.pool_input(1, 4, 3, 3, "negative", 0)
    assert (x < 0).all() and (sc.maxpool3_ref(x) < 0).all()
    zero_pad = F.max_pool2d(F.pad(x.double(), (1, 1, 1, 1)), 3, 2)
    assert (zero_pad == 0).all()
    xi = sc.pool_input(2, 8, 7, 7, "inf", 0)
    assert torch.isposinf(xi).any() and torch.isneginf(xi).any() and not torch.isnan(xi).any()


def test_pool_refs():
    x = sc.pool_input(2, 4, 5, 7, "normal", 3)
    assert sc.maxpool3_out_hw(5, 7) == tuple(sc.maxpool3_ref(x).shape[2:])
    assert sc.maxpool2_ref(x).shape[2:] == (2, 3)
    xd = sc.pool_input(2, 4, 4, 6, "dyadic", 0)
    m, _ = sc.avgpool2_ref(xd)
    assert torch.equal(F.avg_pool2d(xd, 2).double(), m)     # dyadic: exact in float32 too


def test_dwconv_rows():
    assert {(H, W) for _, H, W, *_ in sc.DWCONV_CASES} >= {(1, 5), (6, 1), (1, 1)}
    assert {4, 132} <= {C for _, _, _, C, _, _ in sc.DWCONV_CASES}
    assert {(b, r) for *_, b, r in sc.DWCONV_CASES} == {(False, False), (True, True), (True, False), (False, True)}


def test_dw_convtranspose_rows_and_tap_counts():
    for f in (2, 4, 8):
        rows = [c for c in sc.DWT_CASES if c[4] == f]
        assert {c[5] for c in rows} == {True, False}                            # with and without the addend
        assert any(c[1] == 1 for c in rows)                                     # H = 1
        assert any(c[1] % 2 and c[2] % 2 for c in rows)                         # odd H and W
    for B, H, W, C, f, a in sc.DWT_CASES:
        n = sc.dwt_taps_per_output(H, W, f)
        assert int(n.max()) <= 4                          # gamma(5): at most 4 fmas and the addend
        # every output pixel is reached; the borders by one tap per axis
        assert int(n.min()) >= 1 and int(n[0, 0]) == 1


def test_dw_convtranspose_ref_matches_a_scatter():
    B, H, W, C, f, _ = sc.DWT_CASES[4]
    x, w, a = sc.dwt_operands(B, H, W, C, f, False, "normal", 0)
    want, _ = sc.dwt_ref(x, w, None, f)
    K, pad = 2 * f, f // 2
    out = torch.zeros(B, C, H * f + 2 * K, W * f + 2 * K, dtype=torch.float64)
    for iy in range(H):
        for ix in range(W):
            oy, ox = iy * f - pad + K, ix * f - pad + K
            out[:, :, oy:oy + K, ox:ox + K] += x[:, :, iy, ix, None, None].double() * w[None, :, 0].double()
    assert torch.allclose(out[:, :, K:K + H * f, K:K + W * f], want, rtol=0, atol=1e-12)


def test_copy_rows():
    for (B, H, W), C, in_cs, in_co, out_cs, out_co in sc.COPY_CASES:
        assert C % 4 == 0 and in_co % 4 == 0 and out_co % 4 == 0 and in_cs >= in_co + C and out_cs >= out_co + C


# ---- LookGround ----------------------------------------------------------------------------------------------------------------------
def test_look_ground_flow_is_torch_ports():
    """the restated float32 grid and disparity are exactly what torch_port.look_ground passes to grid_sample"""
    import torch_port as tp
    c = sc.LG_CASES[2]
    g = torch.Generator().manual_seed(0)
    x, _, P2 = sc.lg_inputs(c, 0)
    sd = {"g.disp_create.0.weight": torch.randn(1, c.C, 3, 3, generator=g) * 0.1, "g.disp_create.0.bias": torch.randn(1, generator=g),
          "g.extract.weight": torch.randn(c.C, c.C + 1, 1, 1, generator=g), "g.extract.bias": torch.zeros(c.C), "g.alpha": torch.ones(1)}
    dconv = tp.conv(sd, "g.disp_create.0", x, padding=1)[:, 0]
    seen = {}
    real = tp.F.grid_sample

    def spy(feats, flow, **kw):
        seen["feats"], seen["flow"] = feats.clone(), flow.clone()
        return real(feats, flow, **kw)
    tp.F.grid_sample = spy
    try:
        tp.look_ground(sd, "g", x, P2, baseline=sc.LG_BASELINE, relative_elevation=c.elev)
    finally:
        tp.F.grid_sample = real
    assert torch.equal(seen["flow"], sc.lg_flow(dconv, P2, c.H, c.W, c.elev))
    assert torch.equal(seen["feats"][:, :1], sc.lg_disparity(P2, c.H, c.W, c.elev))


@pytest.mark.parametrize("c", sc.LG_CASES, ids=lambda c: c.name)
def test_look_ground_rows_reach_their_edges(c):
    x, d, P2 = sc.lg_inputs(c, 0)
    flow = sc.lg_flow(d, P2, c.H, c.W, c.elev)
    ix, iy = sc.lg_pixel_coords(flow, c.H, c.W)
    assert c.C % 4 == 0 and c.x_cs % 4 == 0 and c.x_co % 4 == 0 and c.x_cs >= c.x_co + c.C and c.d_cs > c.d_co
    assert len({tuple(P2[b].flatten().tolist()) for b in range(c.B)}) == c.B          # a different camera per image
    if c.name.startswith("integer_grid"):
        assert torch.equal(ix, torch.round(ix)) and torch.equal(iy, torch.round(iy))
        assert torch.equal(iy[0, :, 0], torch.arange(c.H, dtype=torch.float64))       # identity grid
    if c.name.startswith("bottom"):
        assert bool((iy == c.H - 1).any())                 # y1 = H: the bottom row's lower neighbour is out of range
        # some rows pushed below the image before the clip
        raw = (flow[..., 1].double() + 1) / 2 * (c.H - 1)
        assert bool((raw > c.H - 1).any())
    if c.C > 128:
        assert c.C // 4 > 32                               # the warp's channel-quad loop wraps


def test_look_ground_table_covers():
    names = [c.name for c in sc.LG_CASES]
    assert {4, 132} <= {c.C for c in sc.LG_CASES} and (2, 2) in {(c.H, c.W) for c in sc.LG_CASES}
    assert {1.65} < {c.elev for c in sc.LG_CASES}
    assert any(c.x_co > 0 for c in sc.LG_CASES) and any(c.d_co > 0 for c in sc.LG_CASES)
    assert any(n.startswith("integer_grid") for n in names) and any(n.startswith("bottom") for n in names)


@pytest.mark.parametrize("c", sc.LG_CASES, ids=lambda c: c.name)
def test_look_ground_ref_and_bound(c):
    """grid_sample in float64 equals the explicit bilinear; a one-pixel shift or swapped corner weights exceed the bound"""
    x, d, P2 = sc.lg_inputs(c, 0)
    out, S, M = sc.lg_ref(x, d, P2, c.elev)
    flow = sc.lg_flow(d, P2, c.H, c.W, c.elev)
    ix, iy = sc.lg_pixel_coords(flow, c.H, c.W)
    feats = torch.cat([sc.lg_disparity(P2, c.H, c.W, c.elev), x], 1)
    perm = list(range(1, c.C + 1)) + [0]
    assert torch.allclose(sc.bilinear(feats, ix, iy)[:, perm], out, rtol=0, atol=1e-12)
    bound = sc.lg_bound(S, M, c.H, c.W)
    shifted = sc.bilinear(feats, (ix + 1).clamp(max=c.W - 1), iy)[:, perm]
    assert sc.err_ratio(shifted, out, bound) > 100
    shifted = sc.bilinear(feats, ix, (iy - 1).clamp(min=0))[:, perm]
    assert sc.err_ratio(shifted, out, bound) > 100
    if not c.name.startswith("integer_grid") and c.W > 2:
        swapped = sc.bilinear(feats, ix, iy, swap=True)[:, perm]
        assert sc.err_ratio(swapped, out, bound) > 100


# ---- splitters -----------------------------------------------------------------------------------------------------------------------
def _fp16_neighbours(v):
    """the two adjacent fp16 values around float v (as floats) by exhaustive search over positive fp16 bit patterns"""
    allh = torch.arange(0, 0x7C00, dtype=torch.int32).to(torch.int16).view(torch.float16).double()
    a = abs(v)
    lo = float(allh[allh <= a].max())
    hi = float(allh[allh >= a].min())
    return lo, hi


def test_fp16_ties_are_ties_both_ways():
    ups = downs = 0
    for v in sc.fp16_ties():
        assert float(torch.tensor(v, dtype=torch.float64).float()) == v        # exact in float32
        lo, hi = _fp16_neighbours(v)
        assert lo < abs(v) < hi and abs(v) - lo == hi - abs(v)
        r = abs(float(torch.tensor(v).half()))
        lo_bits = int(torch.tensor(lo, dtype=torch.float16).view(torch.int16))
        assert r == (lo if lo_bits % 2 == 0 else hi)                            # round to nearest even
        ups += r == hi
        downs += r == lo
    assert ups > 0 and downs > 0
    assert any(abs(v) < 2.0 ** -14 for v in sc.fp16_ties())                    # subnormal ties


def test_fp16_specials_and_overflows():
    sp = torch.tensor(sc.fp16_specials(), dtype=torch.float64).float()
    assert torch.equal(sp.double(), torch.tensor(sc.fp16_specials(), dtype=torch.float64))
    assert (sp.abs() < sc.FP16_OVERFLOW).all() and torch.isfinite(sp.half()).all()
    assert bool(torch.signbit(sp[1])) and not bool(torch.signbit(sp[0]))         # -0.0 and +0.0
    band = sp[(sp.abs() >= 65504)]
    assert band.numel() >= 4 and torch.equal(band.half().float().abs(), torch.full_like(band, 65504.0))
    assert ((sp.abs() > 0) & (sp.abs() < 2.0 ** -14)).any()                     # fp16 subnormal range
    ov = torch.tensor(sc.fp16_overflows())
    assert (ov.abs() >= sc.FP16_OVERFLOW).all() and torch.isinf(ov.half()).all() and (ov.abs() == sc.FP16_OVERFLOW).any()
    hi, lo = sc.split_h16_ref(sp)
    normal = sp.abs() >= 2.0 ** -14
    assert (lo[normal] != 0).any()                                              # values with bits below the fp16 mantissa


def test_trunc13():
    t = torch.tensor([1.0 + 2.0 ** -23, -3.0 - 2.0 ** -20, 2.0 ** -126, 0.0, -0.0, 2.0 ** 100])
    h = sc.trunc13(t)
    assert torch.equal(h[:2], torch.tensor([1.0, -3.0])) and torch.equal(h[3:], t[3:])
    assert math.isclose(float(t[1] - h[1]), -(2.0 ** -20))
