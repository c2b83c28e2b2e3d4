"""Time the KM3D head's training loss, forward + backward, native (visualdet3d_b200/km3d_loss.py) against the reference's `KM3DHead.loss`
on the same GPU, at the KM3D_example training shape (B = 32, 384x1280 images = 96x320 maps, 3 classes, K = 32) and at B = 8, with the
targets of tests/golden/km3d_loss.npz case a (B = 32 repeats its 8 images 4 times).  Reports ms per step (host clock around steps ending
in a device synchronise: the reference's loss is host-bound), and from one profiled step each: kernel launches, device-to-host copies and
host synchronisations.  The reference arm uses the reference's own compiled iou3d extension (oracle/_ref) when it was built, else the
native one (the record says which), and gets a fresh copy of annotations['dep'] each step because it rewrites it in place.  Prints the
card's name, power limit and max SM clock; writes nothing.

    python tools/bench_km3d_loss.py [--steps 50] [--warmup 10]
The reference arm needs the reference package (oracle/_ref/visualDet3D or the reference tree); without it only the native arm runs."""
import argparse
import importlib.util
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402
from bench_common import card, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    import refload
    from conftest import load_fixture
    from visualdet3d_b200 import _lib, km3d_loss
    spec = importlib.util.spec_from_file_location("gen", os.path.join(ROOT, "tests", "golden", "make_golden_km3d_loss.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    fx = load_fixture("km3d_loss")["a"]
    cfg = km3d_loss.LossConfig(output_w=float(fx["W"]), rampup_length=float(gen.RAMPUP))
    base_out, base_ann = gen.head_outputs(fx), gen.annotations(fx)
    rec = dict(card=card(), torch=torch.__version__, steps=args.steps, warmup=args.warmup, C=int(fx["C"]), H=int(fx["H"]), W=int(fx["W"]),
               K=int(fx["K"]))
    shapes = {}
    for B in (32, 8):
        rep = B // int(fx["B"])
        out = {k: torch.cat([v] * rep).cuda().requires_grad_(True) for k, v in base_out.items()}
        ann = {k: torch.cat([v] * rep).cuda() for k, v in base_ann.items()}
        P2 = torch.from_numpy(fx["P2"]).repeat(rep, 1, 1).cuda()
        shapes[B] = (out, ann, P2)

        def native():
            for t in out.values():
                t.grad = None
            loss, _ = km3d_loss.km3d_head_loss(out, ann, P2, gen.GRAD_EPOCH, cfg)
            loss.backward()

        r = dict(objects=int(ann["reg_mask"].sum()), native=timed(native, args.steps, args.warmup))
        _lib.launch_count_reset()
        native()
        torch.cuda.synchronize()
        r["native"]["native_launches"] = _lib.launch_count()
        rec[f"B{B}"] = r
    if refload.available():
        from visualdet3d_b200.ops import dcn, iou3d
        iou_ext, rec["reference_iou3d"] = iou3d, "native (visualdet3d_b200.ops.iou3d)"
        try:
            import build_ref
            iou_ext, rec["reference_iou3d"] = build_ref.load("ref_iou3d_cuda"), "reference (oracle/_ref ref_iou3d_cuda)"
        except Exception as e:                                   # noqa: BLE001
            rec["reference_iou3d_note"] = f"reference extension unavailable: {e}"
        refload.load_reference(device="cuda", dcn_ext=dcn, iou3d_ext=iou_ext)
        from visualDet3D.networks.heads.km3d_head import KM3DHead
        from visualdet3d_b200.detectors import km3d_cfg
        head = KM3DHead(**refload.to_edict(dict(km3d_cfg().head))).cuda().train()
        for B, (out, ann, P2) in shapes.items():
            def reference():
                for t in out.values():
                    t.grad = None
                loss, _ = head.loss(out, dict(ann, dep=ann["dep"].clone()), dict(P2=P2, epoch=gen.GRAD_EPOCH))
                loss.backward()

            r = rec[f"B{B}"]
            r["reference"] = timed(reference, max(1, args.steps // 5), max(1, args.warmup // 5))
            r["speedup"] = round(r["reference"]["ms_per_step"] / r["native"]["ms_per_step"], 2)
    else:
        rec["reference"] = "not available"
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
