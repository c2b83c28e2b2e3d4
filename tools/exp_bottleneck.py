"""ResNet-101 layer-3 bottleneck convs at the GroundAwareYolo3D shape (batch 8 x 288x1280 -> 18 x 80 x 8 = 11520 pixels): short-K 1x1 convs with wide
outputs.  Tile width sweep (bn_tile) and knock-outs.   python tools/exp_bottleneck.py [reps]"""
import os, sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from visualdet3d_b200 import engine as E

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
B, H, W = 8, 18, 80
g = torch.Generator().manual_seed(0)
planes = lambda C: torch.zeros(2, B, H, W, C, device="cuda", dtype=torch.float16)
flush = torch.empty(64 * 1024 * 1024, device="cuda")


def mk(Cin, Cout, k):
    w = torch.randn(Cout, Cin, k, k, generator=g) / np.sqrt(Cin * k * k)
    return E.ConvLayer(w, torch.randn(Cout, generator=g), None, pad=k // 2, relu=True, device="cuda", engine="tc16")


def act(C):
    return E.split_lo(E.Act(torch.randn(B, H, W, C, generator=g).cuda(), 0, None, planes(C)))


CASES = {"c1 1x1 1024->256": (mk(1024, 256, 1), act(1024), None, 256), "c2 3x3 256->256": (mk(256, 256, 3), act(256), None, 256),
         "c3 1x1 256->1024 +res": (mk(256, 1024, 1), act(256), act(1024), 1024)}


def run(name, label, env, bn, planes_only=False):
    layer, x, res, Cout = CASES[name]
    if planes_only and res is not None:
        res = E.Act(res.t, 0, None, res.lo, f32=False)
    out = E.Act(torch.zeros(B, H, W, Cout, device="cuda"), 0, None, planes(Cout))
    old = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    layer.bn_tile = bn
    try:
        ts = []
        for i in range(reps + 2):
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            layer(x, out, res=res, f32_out=not planes_only)
            b.record()
            torch.cuda.synchronize()
            if i >= 2:
                ts.append(a.elapsed_time(b) * 1e3)
        print(f"{name:24s} {label:44s} median {np.median(ts):8.1f} us  min {min(ts):8.1f}", flush=True)
    except Exception as e:
        print(f"{name:24s} {label:44s} FAILED {e!r}"[:200], flush=True)
    finally:
        layer.bn_tile = 0
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


for name in CASES:
    run(name, "default tile policy", {}, 0)
    for bn in (256, 192, 128, 96, 64):
        run(name, f"bn_tile = {bn}", {}, bn)
    run(name, "default, no epilogue output", {"VD3D_TC_DEBUG": 16}, 0)
    run(name, "default, no residual loads", {"VD3D_TC_DEBUG": 32}, 0)
    run(name, "default, one MMA per k-step", {"VD3D_TC_DEBUG": 1}, 0)
    run(name, "bn 128, no epilogue output", {"VD3D_TC_DEBUG": 16}, 128)
    for bn in (256, 128, 64):
        run(name, f"planes-only output (+ plane residual), bn {bn}", {}, bn, planes_only=True)
