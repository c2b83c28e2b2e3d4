"""Tiles of 80 .. 128 columns run the persistent conv kernel's epilogue on seven dedicated warps, overlapped with the next tile's MMAs;
64-column tiles run it on the consumer warps.  Every output element goes through the same K loop and the same per-element arithmetic
whichever tile width the host picks, so each epilogue-warp width must write exactly what the same conv forced to 64 columns writes: every
bit of the fp32 tensor, both fp16 planes or the tf32 `lo` companion, and the pre-filled sentinels around the written channel slice.

The shapes cover ragged M (Ho * Wo not a multiple of the 128-pixel tile), a last N tile narrower than the tile width, the Cout % 8 == 4
tail, 1 and more than 8 tiles per CTA, every residual form, every output form, and split staging on and off (VD3D_TC_TILE_IN_RING=0).
VD3D_ROW64=0 keeps the 64-column reference on the persistent kernel."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# name: engine, B, Cin, H, W, Cout, k, stride, residual (None / "f32" / "planes"), output ("f32", "planes", "both"), output channel offset
CASES = {
    # 13 x 37 output pixels: partial tiles on both sides; 200 columns leave a narrow last N tile at every width
    "ragged_nores_f32": ("tc16", 2, 128, 13, 37, 200, 3, 1, None, "f32", 4),
    # one 8 x 16 tile: 1 .. 2 tiles per CTA; Cout % 8 == 4 tail
    "one_tile_res_f32_both": ("tc16", 1, 64, 8, 16, 116, 3, 1, "f32", "both", 12),
    "stride2_res_f32_both": ("tc16", 2, 64, 29, 75, 236, 3, 2, "f32", "both", 4),
    # short-K 1x1 expansion conv with a plane residual, planes-only output: 280 M tiles x 2 .. 4 N tiles = 4 .. 9 tiles per CTA
    "shortk_res_planes": ("tc16", 8, 256, 40, 112, 256, 1, 1, "planes", "planes", 8),
    "res_planes_both": ("tc16", 2, 128, 21, 45, 384, 3, 1, "planes", "both", 4),
    "res_planes_f32": ("tc16", 1, 128, 24, 40, 176, 3, 1, "planes", "f32", 4),
    # 3xTF32 engine (vd3d_conv2d_tc): fp32 output alone, and with its tf32 `lo` companion
    "tf32_nores_f32": ("tc", 2, 96, 11, 50, 176, 3, 1, None, "f32", 4),
    "tf32_res_both": ("tc", 2, 64, 17, 50, 240, 3, 1, "f32", "both", 8),
}


def run(name, bn):
    """-> {key: whole output buffer} of case `name` at tile width `bn`"""
    import torch
    sys.path.insert(0, ROOT)
    from visualdet3d_b200 import engine as E
    eng, B, Cin, H, W, Cout, k, s, rmode, oform, co = CASES[name]
    g = torch.Generator().manual_seed(sum(CASES[name][1:8]))
    x = torch.randn(B, H, W, Cin, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / np.sqrt(Cin * k * k)
    b = torch.randn(Cout, generator=g)
    layer = E.ConvLayer(w, b, None, stride=s, pad=k // 2, relu=True, device="cuda", engine=eng)
    assert layer.engine == eng
    layer.bn_tile = bn
    Ho, Wo = layer.out_hw(H, W)
    cs = co + Cout + 8

    def companion(shape, fill):
        if eng == "tc16":
            return torch.full((2,) + shape, fill, device="cuda", dtype=torch.float16)
        return torch.full(shape, fill, device="cuda")

    xa = E.split_lo(E.Act(x.cuda(), 0, None, companion((B, H, W, Cin), 0.0)))
    res = None
    if rmode is not None:
        res = E.split_lo(E.Act(torch.randn(B, Ho, Wo, Cout, generator=g).cuda(), 0, None, companion((B, Ho, Wo, Cout), 0.0)))
        res.f32 = rmode == "f32"
    out = E.Act(torch.full((B, Ho, Wo, cs), 7.0, device="cuda"), co, Cout, None if oform == "f32" else companion((B, Ho, Wo, cs), 3.0))
    layer(xa, out, res=res, f32_out=oform != "planes")
    torch.cuda.synchronize()
    got = {"t": out.t.cpu()}
    if oform != "f32":
        got["planes" if eng == "tc16" else "lo"] = out.lo.cpu()
    return got


@pytest.mark.parametrize("in_ring", [True, False], ids=["ring", "sep_tile"])
@pytest.mark.parametrize("bn", [80, 96, 112, 128])
@pytest.mark.parametrize("name", sorted(CASES))
def test_epilogue_warps_match_consumer_epilogue(name, bn, in_ring, monkeypatch):
    import torch
    monkeypatch.setenv("VD3D_ROW64", "0")
    if not in_ring:
        monkeypatch.setenv("VD3D_TC_TILE_IN_RING", "0")
    ref = run(name, 64)
    got = run(name, bn)
    assert sorted(got) == sorted(ref)
    for key in ref:
        assert torch.equal(got[key], ref[key]), f"{name}: {key} at BN {bn} differs from the 64-column epilogue"
