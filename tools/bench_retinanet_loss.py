"""Time the RetinaNet head's training loss, forward + backward, native (visualdet3d_b200/retina_loss.py) against the reference's
`RetinanetHead.loss` on the same GPU, at RetinaNet_example's training shape (B=8, 288x1280, 3 classes, N = 69210) with 2..12 KITTI-like
boxes per image.  Reports ms per step (host clock around steps ending in a device synchronise: the reference's loss is host-bound), and
from one profiled step each: kernel launches and device-to-host copies / synchronisations.  Prints the card's name and power limit;
writes nothing.

    python tools/bench_retinanet_loss.py [--steps 50] [--warmup 10]
The reference arm needs the reference package (the reference tree or oracle/_ref/visualDet3D); without it only the native arm runs."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
from bench_common import card, timed  # noqa: E402

B, H, W, C, M = 8, 288, 1280, 3, 16


def annotations(seed=0):
    """2..12 boxes per image in the road area, class 0..2, compound_annotation layout (12 columns), padded to M rows."""
    rng = np.random.RandomState(seed)
    ann = np.full((B, M, 12), -1.0, dtype=np.float32)
    for b in range(B):
        for i in range(rng.randint(2, 13)):
            w = rng.uniform(16, 320)
            h = min(w * rng.uniform(0.4, 1.3), H * 0.6)
            x1, y1 = rng.uniform(0, W - w), rng.uniform(H * 0.35, H - h)
            ann[b, i, :5] = [x1, y1, x1 + w, y1 + h, rng.randint(C)]
    return torch.from_numpy(ann).cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    import refload
    from visualdet3d_b200 import retina_loss, synth
    from visualdet3d_b200.anchors import grid_anchors
    hc = synth.retinanet_cfg().head
    a = hc.anchors_cfg
    anchors = torch.from_numpy(grid_anchors((H, W), a["pyramid_levels"], a["strides"], a["sizes"], a["ratios"], a["scales"])
                               .astype(np.float32))[None].cuda()
    N = anchors.shape[1]
    cls, reg = synth.retina_head_outputs(B, N, C, seed=1)
    cls, reg = cls.cuda().requires_grad_(True), reg.cuda().requires_grad_(True)
    ann = annotations()
    cfg = retina_loss.LossConfig.from_loss_cfg(hc.loss_cfg, C, hc.target_means, hc.target_stds)
    rec = dict(B=B, N=N, C=C)

    def native():
        cls.grad = reg.grad = None
        c, r, _ = retina_loss.retinanet_head_loss(cls, reg, anchors, ann, cfg)
        (c + r).backward()

    rec["native"] = timed(native, args.steps, args.warmup)
    if refload.available():
        from visualdet3d_b200.ops import dcn, iou3d
        refload.load_reference(device="cuda", dcn_ext=dcn, iou3d_ext=iou3d)
        from visualDet3D.networks.heads.retinanet_head import RetinanetHead
        head = RetinanetHead(**refload.to_edict(dict(hc, stacked_convs=0, in_channels=8, feat_channels=8))).cuda().train()
        ref_anchors = head.get_anchor(torch.zeros(B, 3, H, W, device="cuda"))
        assert torch.equal(ref_anchors, anchors)

        def reference():
            cls.grad = reg.grad = None
            c, r, _ = head.loss(cls, reg, ref_anchors, ann)
            (c + r).backward()

        rec["reference"] = timed(reference, max(1, args.steps // 5), max(1, args.warmup // 5))
        rec["speedup"] = round(rec["reference"]["ms_per_step"] / rec["native"]["ms_per_step"], 2)
    else:
        rec["reference"] = "not available"
    print(json.dumps(dict(card=card(), torch=torch.__version__, steps=args.steps, warmup=args.warmup, RetinaNet=rec)))


if __name__ == "__main__":
    main()
