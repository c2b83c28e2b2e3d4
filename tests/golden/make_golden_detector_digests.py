"""SHA-256 digests of the six native detectors' inference outputs -> tests/golden/detector_digests.npz: every stage-hook tensor, the kept
rows of the decode outputs (scores, boxes, classes, anchor / peak indices), the per-image counts and the number of library launches per
`launch()`.  Each case is the `build_synthetic_*` detector at seed 0 on two different seeded 96x320 images (B = 2); one more case runs
GroundAwareYolo3D with `post_optimization` and the device post-forward geometry.  The reference comparisons hold the detections to 1e-3,
which a reordered sum or an extra fp16 split passes; the digests pin them bit for bit, so a change to how the detectors are organised must
reproduce them exactly.  Needs a GPU:

    python tests/golden/make_golden_detector_digests.py [--out PATH] [CASE ...]

Recorded from two runs, the second with the cases in reverse order (a different allocator history); only values that agreed are kept.
EXCLUDED names the digests left out for that reason (none: all 97 agreed on an H100).  `tests/test_detector_digests_gpu.py` imports
CASES, EXCLUDED, run_case and record."""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.join(ROOT, "tests", "golden", "detector_digests.npz")
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

B, H, W = 2, 96, 320
CASES = ["Stereo3D", "Yolo3D", "GroundAwareYolo3D", "GroundAwareYolo3D_postopt", "MonoFlex", "KM3D", "RetinaNet"]
EXCLUDED = {}        # case -> keys whose value differed between the two recording runs


def _build(case):
    """-> (detector on cuda, launch arguments on cuda)"""
    from visualdet3d_b200 import synth
    from visualdet3d_b200 import detectors as D
    if case == "Stereo3D":
        det = D.build_synthetic_stereo3d(seed=0)[0]
        left, right, P2, _ = synth.synth_stereo_inputs(B, H, W, seed=1)
        args = (left, right, P2)
    else:
        img, P2 = synth.synth_mono_inputs(B, H, W, seed=1)
        args = (img, P2)
        if case in ("MonoFlex", "KM3D"):
            det = D.build_synthetic_monoflex(seed=0, name=case)[0]
        elif case == "RetinaNet":
            det = D.build_synthetic_retinanet(seed=0)[0]
        else:
            det = D.build_synthetic_mono3d(case.split("_")[0], seed=0)[0]
            det.post_optimization = case.endswith("_postopt")
    return det.cuda().eval(), tuple(a.cuda() for a in args)


def run_case(case):
    """-> {key: output array} of one detector case"""
    import torch
    from visualdet3d_b200 import _lib
    from visualdet3d_b200.engine import Act
    det, args = _build(case)
    got = {}
    with torch.no_grad():
        det.launch(*args)                               # warm-up: folds the plan, sizes the arena, builds the anchor tables
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        det.launch(*args)
        torch.cuda.synchronize()
        got["launches"] = np.array(_lib.launch_count() - n0)
        det.stage_hook = lambda name, v: got.__setitem__(f"stage/{name}", (v.to_nchw() if isinstance(v, Act) else v).detach().cpu().numpy())
        try:
            dec = det.launch(*args)
        finally:
            det.stage_hook = None
        counts = dec.count.tolist()
        got["count"], got["ncand"] = dec.count.cpu().numpy(), dec.ncand.cpu().numpy()
        outs = ["scores", "boxes", "cls", "anchor"]
        if case.endswith("_postopt"):
            P2 = args[-1]
            oP = P2 * torch.tensor([[1.25], [1.25], [1.0]], device=P2.device)     # an original frame 1.25x the network input
            dec.post_forward(P2, oP, corners=True)
            outs += ["box3d", "theta", "box2d", "corners", "homo"]
        for k in outs:
            t = getattr(dec, k)
            got[f"out/{k}"] = np.concatenate([t[b, :n].cpu().numpy().reshape(n, -1) for b, n in enumerate(counts)])
    torch.cuda.synchronize()
    return got


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def record(key, a):
    """what the golden holds for one output: the digest of a stage / decode tensor, the value of a count"""
    return np.array(digest(a)) if key.startswith(("stage/", "out/")) else a


def main(argv):
    out = OUT
    if "--out" in argv:
        i = argv.index("--out")
        out = argv[i + 1]
        del argv[i:i + 2]
    fx = {}
    for case in argv or CASES:
        for key, a in run_case(case).items():
            fx[f"{case}/{key}"] = record(key, a)
            print(case, key, a.dtype, a.shape, fx[f"{case}/{key}"], flush=True)
    np.savez(out, **fx)
    print("wrote", out)


if __name__ == "__main__":
    main(sys.argv[1:])
