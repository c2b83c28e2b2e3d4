"""SHA-256 digests of the persistent tensor-core conv's outputs (fp32 tensor, both fp16 planes or the tf32 `lo` companion, sentinels
included) for seeded inputs -> tests/golden/conv_epilogue.npz.  The digests pin the outputs bit for bit, so a change to how the epilogue is
scheduled (which warps run it, how its loads and stores are mapped) must reproduce them exactly.  Needs a GPU:

    python tests/golden/make_golden_conv_epilogue.py

`tests/test_conv_epilogue_gpu.py` imports CASES and run_case from here."""
import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.join(ROOT, "tests", "golden", "conv_epilogue.npz")

# name: engine, B, Cin, H, W, Cout, k, stride, bn (0: library policy), residual (None / "f32" / "planes"), f32 output, output channel offset
CASES = {
    # the shapes of tests/test_conv_ring_gpu.py
    "bn128": ("tc16", 1, 128, 24, 80, 384, 3, 1, 128, None, True, 4),
    "bn96_res": ("tc16", 2, 128, 24, 80, 384, 3, 1, 96, "f32", True, 4),
    "bn112": ("tc16", 2, 64, 24, 40, 112, 3, 1, 112, None, True, 4),
    "bn64_planes": ("tc16", 3, 64, 40, 112, 64, 3, 1, 64, "planes", False, 4),
    "stride2": ("tc16", 2, 64, 24, 40, 128, 3, 2, 128, None, True, 4),
    "cout72_bn80": ("tc16", 1, 72, 12, 20, 72, 3, 1, 80, "f32", True, 4),
    "ragged608": ("tc16", 3, 64, 24, 48, 608, 3, 1, 128, "f32", True, 4),
    "shortk_1x1": ("tc16", 2, 256, 24, 80, 1024, 1, 1, 64, "planes", False, 4),
    "regtower1408": ("tc16", 8, 1408, 24, 80, 1408, 3, 1, 0, None, True, 4),
    # 1x1 short-K conv (4 k-blocks) with 8 x 6 x 10 x 16 = 7680 tiles, far more than 4 per SM, library tile policy
    "shortk_many_tiles": ("tc16", 8, 256, 48, 160, 1024, 1, 1, 0, "planes", False, 4),
    # ragged last N tile (604 = 4 x 128 + 92: the Cout % 8 == 4 tail) in a channel slice of a wider tensor, sentinels on both sides
    "ragged604_slice": ("tc16", 2, 128, 24, 40, 604, 3, 1, 128, "f32", True, 12),
    # 3xTF32 engine (vd3d_conv2d_tc): fp32 output and its tf32 `lo` companion
    "tf32_out_lo": ("tc", 2, 128, 24, 40, 256, 3, 1, 0, "f32", True, 4),
}


def run_case(name):
    """-> {key: output array} for case `name` (fp32 output `t`; fp16 planes `planes` or tf32 companion `lo`), sentinels included"""
    sys.path.insert(0, ROOT)
    from visualdet3d_b200 import engine as E
    eng, B, Cin, H, W, Cout, k, s, bn, rmode, f32_out, co = CASES[name]
    g = torch.Generator().manual_seed(sum(CASES[name][1:8]))
    x = torch.randn(B, H, W, Cin, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / np.sqrt(Cin * k * k)
    b = torch.randn(Cout, generator=g)
    layer = E.ConvLayer(w, b, None, stride=s, pad=k // 2, relu=True, device="cuda", engine=eng)
    assert layer.engine == eng
    if bn:
        layer.bn_tile = bn
    Ho, Wo = layer.out_hw(H, W)
    cs = co + Cout + 8

    def companion(shape, fill):
        if eng == "tc16":
            return torch.full((2,) + shape, fill, device="cuda", dtype=torch.float16)
        return torch.full(shape, fill, device="cuda")

    xa = E.split_lo(E.Act(x.cuda(), 0, None, companion((B, H, W, Cin), 0.0)))
    res = None
    if rmode is not None:
        res = E.split_lo(E.Act(torch.randn(B, Ho, Wo, Cout, generator=g).cuda(), 0, None, companion((B, Ho, Wo, Cout), 0.0)))
        res.f32 = rmode == "f32"
    out = E.Act(torch.full((B, Ho, Wo, cs), 7.0, device="cuda"), co, Cout, companion((B, Ho, Wo, cs), 3.0))
    layer(xa, out, res=res, f32_out=f32_out)
    torch.cuda.synchronize()
    got = {"planes" if eng == "tc16" else "lo": out.lo.cpu().numpy()}
    if f32_out:
        got["t"] = out.t.cpu().numpy()
    return got


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main():
    fx = {}
    for name in CASES:
        for key, a in run_case(name).items():
            fx[f"{name}/{key}"] = np.array(digest(a))
            print(name, key, a.shape, fx[f"{name}/{key}"], flush=True)
    np.savez(OUT, **fx)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
