"""The 64-channel 3x3 convs of the fp16-split engine run on the row-strip kernel (conv2d_row64.cu).  It must reproduce conv2d_tcp_kernel
(VD3D_ROW64=0) bit for bit: the fp32 output, both fp16 planes, the sentinel channels on both sides of the written channel slice, and the
fp16-range flag, for the same seeded inputs."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# name: B, H, W, Cin, Cout, residual (None / "f32" / "planes"), f32 output, input channel offset, output channel offset, extra environment,
# weight scale (1e5: outputs beyond the fp16 range)
CASES = {
    "layer1": (16, 96, 320, 64, 64, "planes", False, 0, 0, {}, 1.0),
    "layer1_nores": (16, 96, 320, 64, 64, None, False, 0, 0, {}, 1.0),
    "gac": (16, 72, 320, 64, 64, "planes", False, 0, 0, {}, 1.0),
    "dla_f32": (8, 96, 320, 64, 64, "f32", True, 0, 0, {}, 1.0),
    "b1": (1, 96, 320, 64, 64, "planes", True, 0, 0, {}, 1.0),
    "ragged112": (3, 40, 112, 64, 64, "planes", False, 0, 0, {}, 1.0),
    "ragged100": (2, 24, 100, 64, 64, "f32", True, 0, 4, {}, 1.0),
    "odd_h": (2, 25, 72, 64, 64, None, True, 0, 0, {}, 1.0),
    "cout48": (2, 24, 80, 64, 48, "f32", True, 0, 4, {}, 1.0),
    "cin48": (2, 24, 80, 48, 64, "planes", True, 0, 0, {}, 1.0),
    "in_slice": (2, 24, 136, 64, 64, "planes", True, 8, 12, {}, 1.0),
    "chunk2": (4, 48, 160, 64, 64, "planes", False, 0, 0, {"VD3D_TC_CHUNK": "2"}, 1.0),
    "fp16_range": (2, 24, 80, 64, 64, None, True, 0, 0, {}, 1e5),
}


def _run(name, row64, monkeypatch, profile=False):
    from visualdet3d_b200 import engine as E
    B, H, W, Cin, Cout, rmode, f32_out, ci, co, env, scale = CASES[name]
    monkeypatch.setenv("VD3D_ROW64", "1" if row64 else "0")
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    g = torch.Generator().manual_seed(sum((B, H, W, Cin, Cout, ci, co)))
    cs_in = ci + Cin + 8
    x = torch.randn(B, H, W, cs_in, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) * (scale / np.sqrt(Cin * 9))
    b = torch.randn(Cout, generator=g)
    layer = E.ConvLayer(w, b, None, pad=1, relu=rmode is None, device="cuda", engine="tc16")
    assert layer.engine == "tc16"
    xa = E.split_lo(E.Act(x.cuda(), ci, Cin, torch.zeros(2, B, H, W, cs_in, device="cuda", dtype=torch.float16)))
    res = None
    if rmode is not None:
        res = E.split_lo(E.Act(torch.randn(B, H, W, Cout, generator=g).cuda(), 0, None, torch.zeros(2, B, H, W, Cout, device="cuda", dtype=torch.float16)))
        res.f32 = rmode == "f32"
    cs = co + Cout + 8
    out = E.Act(torch.full((B, H, W, cs), 7.0, device="cuda"), co, Cout, torch.full((2, B, H, W, cs), 3.0, device="cuda", dtype=torch.float16))
    E.fp16_range_overflowed(reset=True)
    torch.cuda.synchronize()
    names = set()
    if profile:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            layer(xa, out, res=res, f32_out=f32_out)
            torch.cuda.synchronize()
        names = {e.name for e in prof.events()}
    else:
        layer(xa, out, res=res, f32_out=f32_out)
    torch.cuda.synchronize()
    flag = E.fp16_range_overflowed(reset=True)
    return out.t, out.lo, flag, names


@pytest.mark.parametrize("name", sorted(CASES))
def test_row64_matches_generic_kernel(name, monkeypatch):
    t0, p0, f0, _ = _run(name, False, monkeypatch)
    t1, p1, f1, names = _run(name, True, monkeypatch, profile=name == "layer1")
    if name == "layer1":
        assert any("conv2d_row64_kernel" in n for n in names), sorted(names)
    assert torch.equal(p1.view(torch.int16), p0.view(torch.int16)), f"{name}: fp16 planes differ"
    assert torch.equal(t1.view(torch.int32), t0.view(torch.int32)), f"{name}: fp32 output (or its sentinels) differs"
    assert f1 == f0 and f1 == (name == "fp16_range"), (f0, f1)
