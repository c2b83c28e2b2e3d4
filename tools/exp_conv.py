"""Where does the time of the narrow (64 / 128-channel) tensor-core convs go?  CUDA-event timing of ONE layer shape under the tile-order and
promotion-chunk settings and timing knock-outs (VD3D_TC_DEBUG: results wrong), with fp32 + planes output vs planes-only output / plane residual.
usage: python tools/exp_conv.py [shape] [reps]     shape: layer1 | layer2 | layer3 | head"""
import os, sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from visualdet3d_b200 import engine as E

SHAPES = {"layer1": (16, 96, 320, 64, 64), "layer2": (16, 48, 160, 128, 128), "layer3": (16, 24, 80, 256, 256), "head": (8, 24, 80, 1408, 1408)}
name = sys.argv[1] if len(sys.argv) > 1 else "layer1"
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 20
B, H, W, Cin, Cout = SHAPES[name]
g = torch.Generator().manual_seed(0)
w = torch.randn(Cout, Cin, 3, 3, generator=g) / np.sqrt(Cin * 9)
layer = E.ConvLayer(w, torch.randn(Cout, generator=g), None, pad=1, relu=True, device="cuda", engine="tc16")
planes = lambda C: torch.zeros(2, B, H, W, C, device="cuda", dtype=torch.float16)
x = E.split_lo(E.Act(torch.randn(B, H, W, Cin, generator=g).cuda(), 0, None, planes(Cin)))
res = E.split_lo(E.Act(torch.randn(B, H, W, Cout, generator=g).cuda(), 0, None, planes(Cout)))
res_p = E.Act(res.t, 0, None, res.lo, f32=False)
out = E.Act(torch.zeros(B, H, W, Cout, device="cuda"), 0, None, planes(Cout))
MK = "planes" if Cout <= 160 else "f32"      # mode of the knock-out runs (the widest epilogue variant has no planes form worth timing)
flush = torch.empty(64 * 1024 * 1024, device="cuda")          # 256 MB: evicts the L2 between repetitions


def run(label, env, mode):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        ts = []
        for i in range(reps + 2):
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            if mode == "f32":
                layer(x, out, res=res)
            elif mode == "planes":
                layer(x, out, res=res_p, f32_out=False)
            elif mode == "nores":
                layer(x, out, f32_out=False)
            b.record()
            torch.cuda.synchronize()
            if i >= 2:
                ts.append(a.elapsed_time(b) * 1e3)
        print(f"{name:7s} {label:58s} {mode:7s} median {np.median(ts):8.1f} us  min {min(ts):8.1f}", flush=True)
    except Exception as e:
        print(f"{name:7s} {label:58s} {mode:7s} FAILED {e!r}"[:200], flush=True)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


for mode in ("f32", "planes", "nores"):
    run("default", {}, mode)
for l2 in (0, 28, 44, 64):
    run(f"L2-aware tile order, block = {l2} MB", {"VD3D_TC_L2MB": l2}, "f32")
for dbg, lab in ((16, "knock-out: no epilogue output"), (32, "knock-out: no residual loads"), (48, "knock-out: no output, no residual"),
                 (2, "knock-out: no lo-plane loads"), (1, "knock-out: one MMA per k-step"), (51, "knock-out: 1 MMA, no lo loads, no output, no residual")):
    run(lab, {"VD3D_TC_DEBUG": dbg}, MK)
for dbg, lab in ((64, "knock-out: 1/12 of the MMAs (first K step, one pass), all loads"), (66, "knock-out: 1/12 of the MMAs, no lo loads"),
                 (114, "knock-out: 1/12 MMAs, no lo loads, no output, no residual")):
    run(lab, {"VD3D_TC_DEBUG": dbg}, MK)
for ch in (2, 9, 36):
    run(f"chunk = {ch} k-blocks per promotion", {"VD3D_TC_CHUNK": ch}, MK)
