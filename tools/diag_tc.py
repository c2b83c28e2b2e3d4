"""Diagnostic for the wgmma conv engine: isolates which of the three passes / which k-block pattern is wrong."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch, torch.nn.functional as F
from visualdet3d_b200 import engine as E

def trunc13(t): return (t.contiguous().view(torch.int32) & -8192).view(torch.float32)
def nhwc(x): return x.permute(0, 2, 3, 1).contiguous()

def run(Cin, Cout, k, H=8, W=16, B=1, zero_xlo=False, zero_wlo=False, passes="tc", bn=0):
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / np.sqrt(Cin * k * k)
    layer = E.ConvLayer(w, None, None, pad=k // 2, relu=False, device="cuda", engine=passes)
    if bn: layer.bn_tile = bn
    xa = E.split_lo(E.Act(nhwc(x).cuda(), 0, None, torch.zeros(B, H, W, Cin, device="cuda")))
    if zero_xlo: xa.lo.zero_()
    if zero_wlo: layer.w_lo.zero_()
    out = layer(xa, E.Act(torch.empty(B, H, W, Cout, device="cuda")))
    got = out.to_nchw().cpu().double()
    xh, xl = trunc13(x).double(), trunc13(x - trunc13(x)).double()
    wh, wl = trunc13(w).double(), trunc13(w - trunc13(w)).double()
    if zero_xlo: xl = xl * 0
    if zero_wlo: wl = wl * 0
    conv = lambda a, b: F.conv2d(a, b, padding=k // 2)
    model = conv(xh, wh) + (conv(xl, wh) + conv(xh, wl) if passes == "tc" else 0)
    full = conv(x.double(), w.double())
    e_model = float((got - model).abs().max()); e_full = float((got - full).abs().max())
    e_hh = float((got - conv(xh, wh)).abs().max())
    print(f"Cin={Cin:5d} Cout={Cout:4d} k={k} HxW={H}x{W} zx={int(zero_xlo)} zw={int(zero_wlo)} {passes} bn={layer.bn_tile}: |got-model|={e_model:.2e} |got-fp64|={e_full:.2e} |got-hihi|={e_hh:.2e}")

torch.manual_seed(0)
run(32, 16, 1)
run(64, 16, 1)
run(128, 16, 1)
run(32, 16, 3)
run(64, 64, 3)
run(64, 64, 3, passes="tc1")
run(64, 64, 3, zero_xlo=True)
run(64, 64, 3, zero_wlo=True)
run(64, 64, 3, zero_xlo=True, zero_wlo=True)
run(256, 128, 3, H=24, W=80)
run(256, 128, 3, H=24, W=80, zero_xlo=True)
run(256, 128, 3, H=24, W=80, zero_wlo=True)
run(64, 32, 1, H=24, W=80)
run(64, 64, 1, bn=32)
run(1408, 128, 3, H=24, W=80)
run(1408, 128, 3, H=24, W=80, passes="tc1")
