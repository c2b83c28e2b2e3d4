"""Knock-out timing of the row-strip stem + pool kernel (stem_pool_kernel in csrc/row_conv.cu) at the BASELINE shape (16 images 384x1280):
VD3D_TC_DEBUG bit 0 = one MMA per K step, bit 4 = no output stores.  python tools/exp_stem.py"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from visualdet3d_b200 import engine as E


def main():
    B, H, W = 16, 384, 1280
    g = torch.Generator().manual_seed(0)
    x = torch.randn(B, 3, H, W, generator=g).cuda()
    w = torch.randn(64, 3, 7, 7, generator=g) / np.sqrt(147)
    bn = dict(weight=torch.rand(64, generator=g) + 0.5, bias=torch.randn(64, generator=g) * 0.3,
              running_mean=torch.randn(64, generator=g) * 0.1, running_var=torch.rand(64, generator=g) + 0.5)
    layer = E.StemLayer(w, bn, stride=2, pad=3, relu=True, device="cuda")
    arena = E.Arena("h16")
    out = arena.act("pool", (B, 96, 320, 64), x.device, lo=True)
    lib = E._lib.load()
    Wp, xoff = int(lib.vd3d_stem_pool_row_pitch(W)), int(lib.vd3d_stem_pool_xoff())
    planes = arena.get("rows", (2, B, H, Wp, 4), x.device, dtype=torch.float16, zero=True)
    E.call("vd3d_image_to_h16_rows", x.data_ptr(), B, 3, H, W, planes[0].data_ptr(), planes[1].data_ptr(), Wp, xoff, None)
    oh, ol = out.h16_ptrs

    def run(f32):
        E.call("vd3d_stem_pool_fused", planes[0].data_ptr(), planes[1].data_ptr(), B, H, W, Wp, layer.w_hi.data_ptr(), layer.w_lo.data_ptr(), layer.out_scale,
               layer.b.data_ptr(), out.ptr if f32 else None, oh, ol, out.cs, out.co, None)

    for name, dbg, f32 in [("default (planes only)", 0, False), ("planes + fp32", 0, True), ("one MMA per K step", 1, False), ("no output stores", 16, False),
                           ("one MMA per K step, no output", 17, False)]:
        os.environ["VD3D_TC_DEBUG"] = str(dbg)
        for _ in range(3):
            run(f32)
        ts = []
        for _ in range(20):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            run(f32)
            b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b) * 1e3)
        print(f"stem_pool  {name:36s} median {np.median(ts):8.1f} us  min {min(ts):8.1f}", flush=True)
    os.environ["VD3D_TC_DEBUG"] = "0"


if __name__ == "__main__":
    main()
