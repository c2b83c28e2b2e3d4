"""Time single tensor-core convs of the dominant shapes at several tile widths and check each against the exact-fp32 SIMT engine.
usage: python tools/prof_conv.py [reps] [bns]
  bns: comma list of tile widths (0 = the library's tile policy), e.g. 0,64,128"""
import os, sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from visualdet3d_b200 import engine as E

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
bns = [int(v) for v in (sys.argv[2] if len(sys.argv) > 2 else "0").split(",")]
SHAPES = [("head 1408->1408 @24x80 B8", 8, 24, 80, 1408, 1408, 1), ("layer1 64->64 @96x320 B16", 16, 96, 320, 64, 64, 1),
          ("layer2 128->128 @48x160 B16", 16, 48, 160, 128, 128, 1), ("layer3 256->256 @24x80 B16", 16, 24, 80, 256, 256, 1),
          ("layer2.0 64->128 s2 @96x320 B16", 16, 96, 320, 64, 128, 2), ("odd 72->72 @47x79 B3", 3, 47, 79, 72, 72, 1),
          ("head5 1408->1280 @24x80 B8", 8, 24, 80, 1408, 1280, 1)]
if os.environ.get("PROF_SHAPES"):
    keep = [int(i) for i in os.environ["PROF_SHAPES"].split(",")]
    SHAPES = [SHAPES[i] for i in keep]
g = torch.Generator().manual_seed(0)
cases = []
for name, B, H, W, Cin, Cout, stride in SHAPES:
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / np.sqrt(Cin * 9)
    bias = torch.randn(Cout, generator=g)
    layer = E.ConvLayer(w, bias, None, stride=stride, pad=1, relu=True, device="cuda", engine="tc16")
    ref_layer = E.ConvLayer(w, bias, None, stride=stride, pad=1, relu=True, device="cuda", engine="simt")
    x = E.Act(torch.randn(B, H, W, Cin, generator=g).cuda(), 0, None, torch.zeros(2, B, H, W, Cin, device="cuda", dtype=torch.float16))
    E.split_lo(x)
    Ho, Wo = layer.out_hw(H, W)
    res = E.Act(torch.randn(B, Ho, Wo, Cout, generator=g).cuda())
    ref = ref_layer(E.Act(x.t), E.Act(torch.empty(B, Ho, Wo, Cout, device="cuda")), res=res).t
    torch.cuda.synchronize()
    cases.append((name, B, Ho, Wo, Cin, Cout, layer, 0, x, res, ref))
for bn in bns:
    for name, B, Ho, Wo, Cin, Cout, layer, bn0, x, res, ref in cases:
        layer.bn_tile = bn if bn else bn0
        out = E.Act(torch.zeros(B, Ho, Wo, Cout, device="cuda"), 0, None, torch.zeros(2, B, Ho, Wo, Cout, device="cuda", dtype=torch.float16))
        try:
            layer(x, out, res=res)
            torch.cuda.synchronize()
            err = float((out.t - ref).abs().max())
            hl = float((out.lo[0].float() + out.lo[1].float() - out.t).abs().max())
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                layer(x, out, res=res)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / reps
            clk = ""
            if os.environ.get("PROF_CLOCKS"):       # sustained run (~0.4 s) with nvidia-smi sampling: SM clock under THIS kernel's load
                import importlib.util
                spec = importlib.util.spec_from_file_location("bench", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "bench.py"))
                bench = importlib.util.module_from_spec(spec); spec.loader.exec_module(bench)
                smp = bench.ClockSampler(0); smp.start()
                n = max(20, int(800.0 / ms))
                e0.record()
                for _ in range(n):
                    layer(x, out, res=res)
                e1.record()
                torch.cuda.synchronize()
                c = smp.stop()
                clk = f"  sustained {e0.elapsed_time(e1) / n * 1e3:8.1f} us @ {c['sm_mhz']} MHz {c.get('power_w')} W {c['reasons']}"
            fl = 2.0 * B * Ho * Wo * Cin * Cout * 9
            print(f"{name:34s} bn={layer.bn_tile:3d}  {ms*1e3:8.1f} us  {3*fl/ms/1e9:7.1f} TF/s(x3)  max|err|={err:.2e}  planes={hl:.1e}{clk}", flush=True)
        except Exception as ex:
            print(f"{name:34s} bn={layer.bn_tile:3d}  FAILED: {ex}", flush=True)
            raise SystemExit(1)
