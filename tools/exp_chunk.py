"""Promotion-chunk sweep of the fp16-split conv engine (VD3D_TC_CHUNK = k-blocks accumulated by the tensor core between two promotions into the fp32
registers): error against the REFERENCE fixture at the BASELINE shape (tests/golden/stereo3d_384x1280.npz, the unmodified reference's
outputs on the same seeded inputs) and the step time at batch 8.  The MMA accumulator is updated with truncation (DESIGN 3.1), so longer
chunks are faster (fewer promotion rounds) and less accurate.

    python tools/exp_chunk.py [--chunks 4,6,9,12,18,36]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

from conftest import load_fixture, subsample_like
from visualdet3d_b200 import synth
from visualdet3d_b200.detectors import build_synthetic_stereo3d
from visualdet3d_b200.engine import Act


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", default="4,6,9,12,18,36")
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    det = build_synthetic_stereo3d(seed=0)[0].cuda().eval()
    fx = load_fixture("stereo3d_384x1280")
    H, W, B, seed = [int(v) for v in fx["meta"]]
    left, right, P2, _ = synth.synth_stereo_inputs(B, H, W, seed=1)
    l8, r8, p8, _ = synth.synth_stereo_inputs(8, H, W, seed=1)
    l8, r8, p8 = l8.cuda(), r8.cuda(), p8.cuda()
    for ch in [int(c) for c in args.chunks.split(",")]:
        os.environ["VD3D_TC_CHUNK"] = str(ch)
        st = {}

        def hook(name, v):
            st[name] = v.to_nchw().cpu() if isinstance(v, Act) else v.detach().cpu().clone()
        det.stage_hook = hook
        with torch.no_grad():
            res = det.forward_batch(left.cuda(), right.cuda(), P2.cuda())
        det.stage_hook = None
        st["cls_preds"] = st["cls_preds"].permute(0, 2, 3, 1).reshape(B, -1, det.num_cls_output)
        st["reg_preds"] = st["reg_preds"].permute(0, 2, 3, 1).reshape(B, -1, 12)
        rep = {nm: float(np.abs(subsample_like(st[nm], fx[nm]) - fx[nm]["samples"]).max()) for nm in ["feat4", "features", "cls_preds", "reg_preds"]}
        ds = db = 0.0
        same = True
        for b in range(B):
            s, bx, ci = [t.cpu().numpy() for t in res[b]]
            if len(s) != len(fx[f"scores_{b}"]) or not np.array_equal(ci, fx[f"cls_{b}"]):
                same = False
                continue
            if len(s):
                ds = max(ds, float(np.abs(s - fx[f"scores_{b}"]).max()))
                db = max(db, float(np.abs(bx - fx[f"bboxes_{b}"]).max()))
        with torch.no_grad():
            for _ in range(3):
                det.launch(l8, r8, p8)
            a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            for _ in range(args.steps):
                det.launch(l8, r8, p8)
            e.record()
            torch.cuda.synchronize()
        print(json.dumps({"chunk": ch, "ms_per_step_b8": a.elapsed_time(e) / args.steps, "kept_sets_equal_reference": same,
                          "max_abs_score_err": ds, "max_abs_box_err": db, "stage_max_abs_err": rep}), flush=True)


if __name__ == "__main__":
    main()
