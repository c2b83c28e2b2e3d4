"""SHA-256 digests of the persistent tensor-core conv's outputs (fp32 tensor, both fp16 planes, sentinels included) for seeded inputs whose
ring schedule depends on when the epilogue releases its held stage -> tests/golden/conv_ring_slots.npz.  The producer passes over the held
slot while the epilogue still reads it, and at 112 / 128 columns half the accumulator is staged outside the ring; only buffers and slot
order change, so the outputs must equal the digests recorded with the strictly round-robin ring.  Needs a GPU:

    python tests/golden/make_golden_conv_ring_slots.py

`tests/test_conv_ring_slots_gpu.py` imports CASES and run_case from here.  The inputs are made as in make_golden_conv_epilogue.py."""
import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.join(ROOT, "tests", "golden", "conv_ring_slots.npz")

# name: engine, B, Cin, H, W, Cout, k, stride, bn, residual (None / "f32" / "planes"), f32 output, output channel offset, launch environment
CASES = {
    # BN 128 (3 ring stages) with 1 and 2 k-blocks per tile (1x1, Cin 64 / 128): a tile is over before the held stage comes round again;
    # 3 CTAs, so each runs 40 tiles
    "k1x1_cin64_bn128": ("tc16", 4, 64, 24, 80, 256, 1, 1, 128, "f32", True, 4, {"VD3D_TC_GRID": "3"}),
    "k1x1_cin128_bn128": ("tc16", 4, 128, 24, 80, 256, 1, 1, 128, "planes", True, 4, {"VD3D_TC_GRID": "3"}),
    # long residual epilogues with 60 tiles per CTA: the producer passes over the held slot while the next tile runs
    "res_f32_bn128_grid2": ("tc16", 4, 128, 24, 80, 256, 3, 1, 128, "f32", True, 4, {"VD3D_TC_GRID": "2"}),
    "res_planes_bn128_grid2": ("tc16", 4, 128, 24, 80, 256, 3, 1, 128, "planes", False, 4, {"VD3D_TC_GRID": "2"}),
    # BN 112 (split staging next to 3 stages) with a ragged last N tile (300 = 2 x 112 + 76: the Cout % 8 == 4 tail)
    "bn112_ragged300": ("tc16", 2, 64, 24, 40, 300, 3, 1, 112, "f32", True, 4, {"VD3D_TC_GRID": "4"}),
}


def run_case(name):
    """-> {key: output array} for case `name` (fp32 output `t` when asked, fp16 planes `planes`), sentinels included"""
    sys.path.insert(0, ROOT)
    from visualdet3d_b200 import engine as E
    eng, B, Cin, H, W, Cout, k, s, bn, rmode, f32_out, co, env = CASES[name]
    g = torch.Generator().manual_seed(sum(CASES[name][1:8]))
    x = torch.randn(B, H, W, Cin, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / np.sqrt(Cin * k * k)
    b = torch.randn(Cout, generator=g)
    layer = E.ConvLayer(w, b, None, stride=s, pad=k // 2, relu=True, device="cuda", engine=eng)
    assert layer.engine == eng
    layer.bn_tile = bn
    Ho, Wo = layer.out_hw(H, W)
    cs = co + Cout + 8

    def planes(shape, fill):
        return torch.full((2,) + shape, fill, device="cuda", dtype=torch.float16)

    xa = E.split_lo(E.Act(x.cuda(), 0, None, planes((B, H, W, Cin), 0.0)))
    res = None
    if rmode is not None:
        res = E.split_lo(E.Act(torch.randn(B, Ho, Wo, Cout, generator=g).cuda(), 0, None, planes((B, Ho, Wo, Cout), 0.0)))
        res.f32 = rmode == "f32"
    out = E.Act(torch.full((B, Ho, Wo, cs), 7.0, device="cuda"), co, Cout, planes((B, Ho, Wo, cs), 3.0))
    saved = {key: os.environ.get(key) for key in env}
    os.environ.update(env)
    try:
        layer(xa, out, res=res, f32_out=f32_out)
        torch.cuda.synchronize()
    finally:
        for key, val in saved.items():
            if val is None:
                os.environ.pop(key)
            else:
                os.environ[key] = val
    got = {"planes": out.lo.cpu().numpy()}
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
