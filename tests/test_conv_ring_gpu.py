"""The persistent conv kernel stages its accumulator either in a separate shared-memory tile or in the operand stage of the tile's last k-block
(VD3D_TC_TILE_IN_RING, default 1: one more stage of operand ring).  Only buffers move: the MMAs and the epilogue are the same, so both forms
must give the same bits -- fp32 output and both fp16 planes -- for every tile width, stride, output form and tile order."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _E():
    from visualdet3d_b200 import engine
    return engine


def _planes(*shape, fill=0.0):
    return torch.full((2,) + shape, fill, device="cuda", dtype=torch.float16)


CASES = [
    # B, Cin, H, W, Cout, k, stride, bn, residual (None / "f32" / "planes"), f32 output
    (1, 128, 24, 80, 384, 3, 1, 128, None, True),         # 128-column tiles: unpadded, swizzled staging rows
    (2, 128, 24, 80, 384, 3, 1, 96, "f32", True),
    (2, 64, 24, 40, 112, 3, 1, 112, None, True),          # 112 columns: padded rows, 2 -> 3 stages
    (3, 64, 40, 112, 64, 3, 1, 64, "planes", False),      # planes-only output and a plane residual, more tiles than SMs
    (2, 64, 24, 40, 128, 3, 2, 128, None, True),          # stride 2
    (1, 72, 12, 20, 72, 3, 1, 80, "f32", True),           # ragged Cout inside an 80-column tile
    (3, 64, 24, 48, 608, 3, 1, 128, "f32", True),         # ragged last N tile (608 = 4 x 128 + 96)
    (2, 256, 24, 80, 1024, 1, 1, 64, "planes", False),    # short K (4 k-blocks): the held stage comes round every tile
    (8, 1408, 24, 80, 1408, 3, 1, 0, None, True),         # the reg-tower conv: L2-blocked tile order, default tile policy
]


def _run(layer, xa, res, B, Ho, Wo, Cout, f32_out):
    E = _E()
    out = E.Act(torch.full((B, Ho, Wo, Cout + 8), 7.0, device="cuda"), 4, Cout, _planes(B, Ho, Wo, Cout + 8, fill=3.0))
    layer(xa, out, res=res, f32_out=f32_out)
    torch.cuda.synchronize()
    return out.t.clone(), out.lo.clone()


@pytest.mark.parametrize("case", CASES)
def test_staging_in_ring_is_bit_identical(case, monkeypatch):
    E = _E()
    B, Cin, H, W, Cout, k, s, bn, rmode, f32_out = case
    g = torch.Generator().manual_seed(sum(case[:7]))
    x = torch.randn(B, H, W, Cin, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / np.sqrt(Cin * k * k)
    b = torch.randn(Cout, generator=g)
    layer = E.ConvLayer(w, b, None, stride=s, pad=k // 2, relu=True, device="cuda", engine="tc16")
    assert layer.engine == "tc16"
    layer.bn_tile = bn
    Ho, Wo = layer.out_hw(H, W)
    xa = E.split_lo(E.Act(x.cuda(), 0, None, _planes(B, H, W, Cin)))
    res = None
    if rmode is not None:
        res = E.split_lo(E.Act(torch.randn(B, Ho, Wo, Cout, generator=g).cuda(), 0, None, _planes(B, Ho, Wo, Cout)))
        res.f32 = rmode == "f32"
    got = {}
    for ring in ("0", "1"):
        monkeypatch.setenv("VD3D_TC_TILE_IN_RING", ring)
        got[ring] = _run(layer, xa, res, B, Ho, Wo, Cout, f32_out)
    (t0, p0), (t1, p1) = got["0"], got["1"]
    assert torch.equal(p0, p1), case
    if f32_out:
        assert torch.equal(t0, t1), case
        hi = t1[..., 4:4 + Cout].half()
        assert torch.equal(p1[0][..., 4:4 + Cout], hi)
    assert float(p1[..., :4].float().min()) == 3.0 and float(p1[..., 4 + Cout:].float().min()) == 3.0
    assert float(t1[..., :4].min()) == 7.0 and float(t1[..., 4 + Cout:].min()) == 7.0


def test_staging_in_ring_stem_pool_is_bit_identical(monkeypatch):
    """the 8 x 16-tile stem with the fused max-pool (16-pixel windows on 128-byte rows: 64-column tiles whose pool epilogue reads the staged
    tile with its own row pitch)"""
    E = _E()
    monkeypatch.setenv("VD3D_STEM_WIN", "64")
    g = torch.Generator().manual_seed(5)
    B, C, H, W = 2, 3, 96, 320
    x = (torch.randn(B, C, H, W, generator=g) * 2.0).cuda()
    w = torch.randn(64, C, 7, 7, generator=g) / np.sqrt(C * 49)
    bn = dict(weight=torch.rand(64, generator=g) + 0.5, bias=torch.randn(64, generator=g) * 0.3,
              running_mean=torch.randn(64, generator=g) * 0.1, running_var=torch.rand(64, generator=g) + 0.5)
    layer = E.StemLayer(w, bn, stride=2, pad=3, relu=True, device="cuda")
    assert not layer.row_kernel_ok()
    Hs, Ws = layer.out_hw(H, W)
    Hp, Wp = (Hs - 1) // 2 + 1, (Ws - 1) // 2 + 1
    arena = E.Arena("h16")
    got = {}
    for ring in ("0", "1"):
        monkeypatch.setenv("VD3D_TC_TILE_IN_RING", ring)
        out = E.Act(torch.full((B, Hp, Wp, 64), 7.0, device="cuda"))
        layer(x, out, arena, "p", pool=True)
        full = layer(x, E.Act(torch.empty(B, Hs, Ws, 64, device="cuda")), arena, "f")
        torch.cuda.synchronize()
        got[ring] = (out.t.clone(), full.t.clone())
    assert torch.equal(got["0"][0], got["1"][0]) and torch.equal(got["0"][1], got["1"][1])
    assert float(got["1"][0].min()) >= 0.0 and float((got["1"][0] == 0).float().mean()) < 0.9
