"""Step-form timing of the backbone's 64 -> 64 3x3 convs (ResNet layer1 and its kin): fp16-plane input, plane residual or none, planes-only
output, as the stereo step runs them.  CUDA events around `reps` back-to-back launches (after a warm-up), repeated; the median per launch is
printed for every engine setting and timing knock-out (VD3D_TC_DEBUG: results wrong), together with the card name, power limit, SM clock and
board power read while a burst of the same conv runs.
usage: python tools/exp_layer1.py [shape ...] [--reps N] [--quick]      shape: layer1 (default) | gac"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from visualdet3d_b200 import engine as E

SHAPES = {"layer1": (16, 96, 320), "gac": (16, 72, 320)}
C = 64
TC_FLOOR_CLK = 201e3          # tensor clocks per SM of one layer1 conv (3 products, 108.7 GFLOP over 132 SMs)

# (label, environment): the production kernel, the generic kernel, and the generic kernel's knock-outs
CONFIGS = [
    ("production", {}),
    ("generic kernel (VD3D_ROW64=0)", {"VD3D_ROW64": 0}),
    ("generic, no lo-plane loads (DEBUG=2)", {"VD3D_ROW64": 0, "VD3D_TC_DEBUG": 2}),
    ("generic, no epilogue output (DEBUG=16)", {"VD3D_ROW64": 0, "VD3D_TC_DEBUG": 16}),
    ("generic, no residual loads (DEBUG=32)", {"VD3D_ROW64": 0, "VD3D_TC_DEBUG": 32}),
    ("generic, no lo loads + no output (DEBUG=18)", {"VD3D_ROW64": 0, "VD3D_TC_DEBUG": 18}),
    ("generic, 66 CTAs (VD3D_TC_GRID=66)", {"VD3D_ROW64": 0, "VD3D_TC_GRID": 66}),
    ("row kernel, no epilogue output (DEBUG=16)", {"VD3D_TC_DEBUG": 16}),
]


def smi(fields):
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as e:       # (reported, not fatal: the timing stands without it)
        return f"nvidia-smi unavailable: {e!r}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("shapes", nargs="*", default=["layer1"])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--quick", action="store_true", help="production vs generic only")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "exp_layer1 needs a GPU"
    print("card:", smi("name,power.limit,clocks.max.sm"), flush=True)
    g = torch.Generator().manual_seed(0)
    for shape in a.shapes:
        B, H, W = SHAPES[shape]
        w1 = torch.randn(C, C, 3, 3, generator=g) / np.sqrt(C * 9)
        layer = E.ConvLayer(w1, torch.randn(C, generator=g), None, pad=1, relu=True, device="cuda", engine="tc16")
        planes = lambda: torch.zeros(2, B, H, W, C, device="cuda", dtype=torch.float16)
        x = E.split_lo(E.Act(torch.randn(B, H, W, C, generator=g).cuda(), 0, None, planes()))
        r = E.split_lo(E.Act(torch.randn(B, H, W, C, generator=g).cuda(), 0, None, planes()))
        res_p = E.Act(r.t, 0, None, r.lo, f32=False)
        out = E.Act(torch.zeros(B, H, W, C, device="cuda"), 0, None, planes())
        floor_us = TC_FLOOR_CLK * (B * H * W) / (16 * 96 * 320) / 1275.0
        print(f"== {shape}: 64 -> 64 3x3 @ {H}x{W}, B {B}; three-product tensor floor ~{floor_us:.0f} us at 1275 MHz", flush=True)
        for label, env in (CONFIGS[:2] if a.quick else CONFIGS):
            old = {k: os.environ.get(k) for k in env}
            os.environ.update({k: str(v) for k, v in env.items()})
            try:
                for mode in ("nores", "planes"):
                    call = (lambda: layer(x, out, f32_out=False)) if mode == "nores" else (lambda: layer(x, out, res=res_p, f32_out=False))
                    for _ in range(3):
                        call()
                    torch.cuda.synchronize()
                    ts = []
                    for _ in range(a.rounds):
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        for _ in range(a.reps):
                            call()
                        e1.record()
                        torch.cuda.synchronize()
                        ts.append(e0.elapsed_time(e1) * 1e3 / a.reps)
                    clk = ""
                    if label == "production" or mode == "planes" and label.startswith("generic kernel"):
                        for _ in range(600):       # a burst of ~0.2 s: clocks and board power under this load
                            call()
                        clk = "  [" + smi("clocks.sm,power.draw") + "]"
                        torch.cuda.synchronize()
                    print(f"{shape:7s} {label:46s} {'residual' if mode == 'planes' else 'no res':8s} median {np.median(ts):7.1f} us  "
                          f"min {min(ts):7.1f}{clk}", flush=True)
            finally:
                for k, v in old.items():
                    if v is None:
                        os.environ.pop(k, None)
                    else:
                        os.environ[k] = v


if __name__ == "__main__":
    main()
