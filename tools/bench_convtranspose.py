"""Kernel time of the three transposed convs of the ResNet-18 CenterNet core (KM3D_example) at batch 8, 384x1280, on the fp16-split engine
(vd3d_convtranspose2d_tc16: four sub-pixel 2x2 phase convs in one launch), against F.conv_transpose2d in fp32 on the same card.

    python tools/bench_convtranspose.py [iters] [repeats]     -> one JSON line per layer

Per layer: CUDA events around `iters` back-to-back launches, `repeats` times (median, min, max ms per launch), after a warm-up.  FLOP
are the layer's own (2 x B x 2H x 2W x Cout x Cin x 4 taps: the 4x4 kernel at stride 2 touches 4 taps per output pixel); the MMA floor
is the engine's three fp16 products per MAC at the data sheet's dense FP16 rate (989 TFLOP/s, H100 SXM at 700 W)."""
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_common import card  # noqa: E402
from visualdet3d_b200 import engine as E  # noqa: E402

FP16_DENSE_TFLOPS = 989.0
B, H0, W0 = 8, 384, 1280
LAYERS = [(512, 256, H0 // 32, W0 // 32), (256, 256, H0 // 16, W0 // 16), (256, 256, H0 // 8, W0 // 8)]    # (Cin, Cout, input H, W)


def time_ms(fn, iters, repeats):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / iters)
    out.sort()
    return out[len(out) // 2], out[0], out[-1]


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 50
    repeats = int(sys.argv[2]) if len(sys.argv) > 2 else 7
    if not torch.cuda.is_available():
        raise SystemExit("bench_convtranspose: needs a GPU")
    dev = torch.device("cuda")
    gpu = card()
    g = torch.Generator().manual_seed(0)
    for i, (Cin, Cout, H, W) in enumerate(LAYERS):
        wt = torch.randn(Cin, Cout, 4, 4, generator=g) * (2.0 / (4 * Cin)) ** 0.5
        bn = dict(weight=torch.rand(Cout, generator=g) + 0.5, bias=torch.randn(Cout, generator=g) * 0.1,
                  running_mean=torch.randn(Cout, generator=g) * 0.1, running_var=torch.rand(Cout, generator=g) + 0.5)
        layer = E.ConvTransposeLayer(wt, bn, relu=True, device=dev)
        x = torch.randn(B, H, W, Cin, device=dev)
        xa = E.split_lo(E.Act(x, 0, None, torch.zeros((2, B, H, W, Cin), dtype=torch.float16, device=dev)))
        out = E.Act(torch.empty(B, 2 * H, 2 * W, Cout, device=dev), 0, None, torch.zeros((2, B, 2 * H, 2 * W, Cout), dtype=torch.float16, device=dev))
        with torch.no_grad():
            planes = time_ms(lambda: layer(xa, out, f32_out=False), iters, repeats)
            both = time_ms(lambda: layer(xa, out, f32_out=True), iters, repeats)
            xn = x.permute(0, 3, 1, 2).contiguous()
            wd = wt.to(dev)
            torch.backends.cudnn.allow_tf32 = False
            ref = time_ms(lambda: F.conv_transpose2d(xn, wd, None, stride=2, padding=1), iters, repeats)
        flop = 2.0 * B * (2 * H) * (2 * W) * Cout * Cin * 4
        floor_ms = 3 * flop / (FP16_DENSE_TFLOPS * 1e12) * 1e3
        print(json.dumps({"layer": f"deconv_layers.{3 * i}", "shape": f"{Cin}->{Cout}, {B}x{H}x{W} -> {2 * H}x{2 * W}", "gflop": round(flop / 1e9, 2),
                          "planes_only_ms": [round(v, 4) for v in planes], "fp32_and_planes_ms": [round(v, 4) for v in both],
                          "tflops_planes_only": round(flop / (planes[0] * 1e-3) / 1e12, 1),
                          "mma_floor_share": round(floor_ms / planes[0], 3),
                          "torch_conv_transpose2d_fp32_ms": [round(v, 4) for v in ref],
                          "timing": f"median, min, max of {repeats} x {iters} launches (CUDA events)", "card": gpu}), flush=True)


if __name__ == "__main__":
    main()
