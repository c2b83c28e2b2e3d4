"""SHA-256 digests of the row-strip kernels' outputs -> tests/golden/row_strip_digests.npz: `vd3d_row_conv` (fp32 and plane outputs,
and the planes of a planes-only call) on every `ROW_CONV_CASES` entry of tests/test_ops_gpu.py, `vd3d_stem_pool_fused` (pooled planes,
with and without the fp32 output) at the shapes of `test_stem_row_strip_kernel_is_bit_identical`, and the row planes written by
`vd3d_image_to_h16_rows` and `vd3d_image_to_h16_rows_c` (4 and 8 channels per pixel).  `test_row_conv_vs_fp64` allows 2e-5, which a
reordered MMA chain passes; the digests pin every output bit, whole buffers included (borders and neighbouring channels), so a change to
how the row-strip kernels are organised must reproduce them exactly.  Needs a GPU:

    python tests/golden/make_golden_row_strip_digests.py [--out PATH] [CASE ...]

Recorded from two runs, the second with the cases in reverse order (a different allocator history); only values that agreed are kept.
EXCLUDED names the digests left out for that reason (none on an H100).  `tests/test_row_strip_digests_gpu.py` imports CASES, EXCLUDED,
run_case and digest."""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.join(ROOT, "tests", "golden", "row_strip_digests.npz")
for _p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from test_ops_gpu import ROW_CONV_CASES  # noqa: E402

STEM_SHAPES = [(2, 3, 64, 96), (3, 3, 70, 154), (1, 3, 34, 30), (2, 3, 96, 320), (16, 3, 96, 160), (2, 3, 384, 1280), (1, 3, 75, 515), (5, 3, 21, 1010)]
PLANE_CASES = [("rows", 3, 4), ("rows", 4, 4), ("rows_c", 3, 4), ("rows_c", 4, 4), ("rows_c", 3, 8), ("rows_c", 8, 8)]   # entry, C, cpad

CASES = ([f"row_conv/{'_'.join(map(str, c))}" for c in ROW_CONV_CASES]
         + [f"stem/{'_'.join(map(str, s))}/{'f32' if f else 'planes'}" for s in STEM_SHAPES for f in (True, False)]
         + [f"planes/{e}/c{c}/p{p}" for e, c, p in PLANE_CASES])
EXCLUDED = {}        # case -> keys whose value differed between the two recording runs


def _row_conv(case):
    """the inputs, layer and output buffers of test_row_conv_vs_fp64"""
    import torch
    from visualdet3d_b200 import engine as E
    B, Cin, pc, H, W, Cout, k, s, p = case
    g = torch.Generator().manual_seed(sum(case))
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / np.sqrt(Cin * k * k)
    bn = dict(weight=torch.rand(Cout, generator=g) + 0.5, bias=torch.randn(Cout, generator=g) * 0.3,
              running_mean=torch.randn(Cout, generator=g) * 0.1, running_var=torch.rand(Cout, generator=g) + 0.5)
    layer = E.RowConvLayer(w, bn, stride=s, pad=p, relu=True, pc_in=pc, device="cuda")
    xoff = p + (2 if pc == 4 else 1)
    Wp = layer.in_pitch(W, xoff)
    planes = torch.zeros(2, B, H, Wp, pc, dtype=torch.float16, device="cuda")
    if Cin <= 4 and pc in (4, 8):
        xin = E.image_to_row_planes(x.cuda(), planes, xoff)
    else:
        xh = x.half()
        xl = (x - xh.float()).half()
        planes[0, :, :, xoff:xoff + W, :Cin] = xh.permute(0, 2, 3, 1).cuda()
        planes[1, :, :, xoff:xoff + W, :Cin] = xl.permute(0, 2, 3, 1).cuda()
        xin = E.RowPlanes(planes, W, xoff)
    Ho, Wo = layer.out_hw(H, W)
    oW, oxo, cs, co = Wo + 5, 2, Cout + 16, 8
    of = torch.full((B, Ho, oW, cs), 7.0, device="cuda")
    op = torch.full((2, B, Ho, oW, cs), 3.0, device="cuda", dtype=torch.float16)
    layer(xin, op, of, out_xoff=oxo, out_co=co)
    op2 = torch.full_like(op, 3.0)
    layer(xin, op2, None, out_xoff=oxo, out_co=co)
    return dict(out_f32=of, out_planes=op, planes_only=op2)


def _stem(shape, f32_out):
    """the inputs, layer and output buffers of test_stem_row_strip_kernel_is_bit_identical"""
    import torch
    from visualdet3d_b200 import engine as E
    B, C, H, W = shape
    g = torch.Generator().manual_seed(sum(shape))
    x = (torch.randn(B, C, H, W, generator=g) * 2.0).cuda()
    w = torch.randn(64, C, 7, 7, generator=g) / np.sqrt(C * 49)
    bn = dict(weight=torch.rand(64, generator=g) + 0.5, bias=torch.randn(64, generator=g) * 0.3,
              running_mean=torch.randn(64, generator=g) * 0.1, running_var=torch.rand(64, generator=g) + 0.5)
    layer = E.StemLayer(w, bn, stride=2, pad=3, relu=True, device="cuda")
    assert layer.row_kernel_ok()
    Hs, Ws = layer.out_hw(H, W)
    Hp, Wp = (Hs - 1) // 2 + 1, (Ws - 1) // 2 + 1
    got = E.Act(torch.full((B, Hp, Wp, 64 + 16), 7.0, device="cuda"), 8, 64, torch.full((2, B, Hp, Wp, 64 + 16), 3.0, device="cuda", dtype=torch.float16))
    layer(x, got, E.Arena("h16"), "b", pool=True, f32_out=f32_out)
    assert layer.wrote_planes
    return dict(out_f32=got.t, out_planes=got.lo)


def _planes(entry, C, cpad):
    """an image (with channels beyond C, image columns beyond W and pixels in front of xoff left as they were) -> row planes"""
    import torch
    from visualdet3d_b200._lib import call
    B, H, W, xoff = 2, 37, 53, 5
    g = torch.Generator().manual_seed(C * 16 + cpad)
    x = (torch.randn(B, C, H, W, generator=g) * 3.0).cuda()
    Wp = W + xoff + 7
    planes = torch.full((2, B, H, Wp, cpad), 3.0, device="cuda", dtype=torch.float16)
    if entry == "rows":
        call("vd3d_image_to_h16_rows", x.data_ptr(), B, C, H, W, planes[0].data_ptr(), planes[1].data_ptr(), Wp, xoff, None)
    else:
        call("vd3d_image_to_h16_rows_c", x.data_ptr(), B, C, H, W, planes[0].data_ptr(), planes[1].data_ptr(), Wp, xoff, cpad, None)
    return dict(planes=planes)


def run_case(case):
    """-> {key: output array} of one case"""
    import torch
    kind, rest = case.split("/", 1)
    if kind == "row_conv":
        got = _row_conv(tuple(int(v) for v in rest.split("_")))
    elif kind == "stem":
        shape, out = rest.split("/")
        got = _stem(tuple(int(v) for v in shape.split("_")), out == "f32")
    else:
        entry, c, p = rest.split("/")
        got = _planes(entry, int(c[1:]), int(p[1:]))
    torch.cuda.synchronize()
    return {k: v.detach().cpu().numpy() for k, v in got.items()}


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main(argv):
    out = OUT
    if "--out" in argv:
        i = argv.index("--out")
        out = argv[i + 1]
        del argv[i:i + 2]
    fx = {}
    for case in argv or CASES:
        for key, a in run_case(case).items():
            fx[f"{case}/{key}"] = np.array(digest(a))
            print(case, key, a.dtype, a.shape, fx[f"{case}/{key}"], flush=True)
    np.savez(out, **fx)
    print("wrote", out)


if __name__ == "__main__":
    main(sys.argv[1:])
