"""Time the 3-D anchor head's training loss, forward + backward, native (visualdet3d_b200/anchor_loss.py) against the reference's
`AnchorBasedDetection3DHead.loss` on the same GPU, at the training shapes of Stereo3D (B=4, 288x1280, 2 classes, N = 69120) and
GroundAwareYolo3D (B=8, 288x1280, 1 class, N = 46080).  Reports ms per step (host clock around steps ending in a device synchronise:
the reference's loss is host-bound), and from one profiled step each: kernel launches and device-to-host copies / synchronisations.
Prints the card's name and power limit; writes nothing.

    python tools/bench_anchor_loss.py [--steps 50] [--warmup 10]
The reference arm needs the reference package (the reference tree or oracle/_ref/visualDet3D); without it only the native arm runs."""
import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
from bench_common import card, timed  # noqa: E402

SHAPES = {"Stereo3D": dict(B=4, kind="Stereo3D"), "GroundAwareYolo3D": dict(B=8, kind="GroundAwareYolo3D")}
H, W, M = 288, 1280, 8


def annotations(B, C, seed=0):
    """Six ground truths per image in the road area of the image, compound_annotation layout, padded to M rows."""
    rng = np.random.RandomState(seed)
    ann = np.full((B, M, 12), -1.0, dtype=np.float32)
    for b in range(B):
        for i in range(6):
            w = rng.uniform(24, 300)
            h = min(w * rng.uniform(0.4, 1.3), H * 0.6)
            x1, y1 = rng.uniform(0, W - w), rng.uniform(H * 0.35, H - h)
            ann[b, i] = [x1, y1, x1 + w, y1 + h, rng.randint(C), x1 + w / 2, y1 + h / 2, rng.uniform(5, 50), 1.6, 1.5, 3.9,
                         rng.uniform(-np.pi, np.pi)]
    return torch.from_numpy(ann).cuda()


def setup(name, ref_head_cls):
    from visualdet3d_b200 import synth
    from visualdet3d_b200.anchors import AnchorTable
    kind, B = SHAPES[name]["kind"], SHAPES[name]["B"]
    tmp = tempfile.mkdtemp()
    obj_types = ["Car"] if kind == "GroundAwareYolo3D" else ["Car", "Pedestrian"]
    pm, ps = synth.synth_priors(16, 2 if len(obj_types) == 1 else 3, obj_types)
    synth.write_priors(tmp, pm, ps, obj_types)
    hc = synth.mono3d_cfg(tmp, kind).head if kind == "GroundAwareYolo3D" else synth.stereo3d_cfg(tmp).head
    C = len(obj_types)
    P2 = synth.synth_P2(B, H, W)[0].cuda()
    head = None
    if ref_head_cls is not None:
        import refload
        layer = dict(num_features_in=8, num_cls_output=C + 1, num_reg_output=12, cls_feature_size=8, reg_feature_size=8)
        head = ref_head_cls(num_features_in=8, num_classes=C, num_regression_loss_terms=13, preprocessed_path=tmp,
                            anchors_cfg=refload.to_edict(dict(hc.anchors_cfg)), layer_cfg=refload.to_edict(layer),
                            loss_cfg=refload.to_edict(dict(hc.loss_cfg)), test_cfg=refload.to_edict(dict(hc.test_cfg))).cuda().train()
        anchors = head.get_anchor(torch.zeros(B, 3, H, W, device="cuda"), P2)
    else:
        table = AnchorTable((H, W), hc.anchors_cfg, pm, ps, "cuda")
        anchors = dict(anchors=table.anchors[None], mask=torch.ones(B, table.N, dtype=torch.bool, device="cuda"),
                       anchor_mean_std_3d=table.mean_std)
    N = anchors["anchors"].shape[1]
    cls, reg = synth.synth_head_outputs(B, N, C, seed=1)
    return head, hc.loss_cfg, anchors, annotations(B, C), P2, cls.cuda().requires_grad_(True), reg.cuda().requires_grad_(True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    import refload
    from visualdet3d_b200 import anchor_loss
    ref_cls = None
    if refload.available():
        from visualdet3d_b200.ops import dcn, iou3d
        refload.load_reference(device="cuda", dcn_ext=dcn, iou3d_ext=iou3d)
        from visualDet3D.networks.heads.detection_3d_head import AnchorBasedDetection3DHead
        ref_cls = AnchorBasedDetection3DHead
    out = dict(card=card(), torch=torch.__version__, steps=args.steps, warmup=args.warmup, shapes={})
    for name in SHAPES:
        head, loss_cfg, anchors, ann, P2, cls, reg = setup(name, ref_cls)
        cfg = anchor_loss.LossConfig.from_loss_cfg(loss_cfg, cls.shape[-1] - 1)
        rec = dict(B=cls.shape[0], N=cls.shape[1], C=cls.shape[2] - 1)

        def native():
            cls.grad = reg.grad = None
            c, r, _ = anchor_loss.anchor3d_head_loss(cls, reg, anchors, ann, cfg)
            (c + r).sum().backward()

        rec["native"] = timed(native, args.steps, args.warmup)
        if head is not None:
            def reference():
                cls.grad = reg.grad = None
                c, r, _ = head.loss(cls, reg, anchors, ann, P2)
                (c + r).sum().backward()

            rec["reference"] = timed(reference, max(1, args.steps // 5), max(1, args.warmup // 5))
            rec["speedup"] = round(rec["reference"]["ms_per_step"] / rec["native"]["ms_per_step"], 2)
        else:
            rec["reference"] = "not available"
        out["shapes"][name] = rec
    print(json.dumps(out))


if __name__ == "__main__":
    main()
