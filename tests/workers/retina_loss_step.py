"""Worker of tests/test_retina_loss_gpu.py::test_reference_{head,detector}_training_step (own process, GPU box).

    retina_loss_step.py head       one training step of the reference's UNMODIFIED RetinanetHead (RetinaNet_example head: 4 stacked
                                   256-channel convs over 256-channel P3..P7 features, 3 classes) at B=8, 288x1280
    retina_loss_step.py detector   one training step of the reference's RetinaNet (ResNet-50 + FPN + head, pretrained=False) through
                                   `RetinaNet([img, annotations, calib])` at B=2, 96x320

each first with the reference's own Python loss, then with `plugin.install_retinanet_loss_into_reference()` in place: the same inputs
and annotations (tests/golden/retina_loss.npz, packed into an odd row count).  The zero-initialised output convs get small seeded weights, so gradients reach the
layers below them.  Prints one JSON line with the loss and parameter-gradient differences."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import refload  # noqa: E402


def main(mode):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False
    from visualdet3d_b200.ops import dcn as our_dcn, iou3d as our_iou
    from visualdet3d_b200 import plugin, retina_loss, synth
    refload.load_reference(device="cuda", dcn_ext=our_dcn, iou3d_ext=our_iou)
    from visualDet3D.networks.heads.retinanet_head import RetinanetHead
    from visualDet3D.networks.detectors.retinanet_2d import RetinaNet

    fx = np.load(os.path.join(ROOT, "tests", "golden", "retina_loss.npz"))

    def odd_rows(ann):
        """The valid rows in their order, packed into the smallest odd row count holding them, as a trainer's padding often leaves them."""
        valid = ann[:, :, 4] != -1
        out = np.full((ann.shape[0], int(valid.sum(1).max()) | 1, ann.shape[2]), -1.0, dtype=np.float32)
        for b in range(ann.shape[0]):
            out[b, :valid[b].sum()] = ann[b][valid[b]]
        return out

    cfg = refload.to_edict(dict(synth.retinanet_cfg()))
    torch.manual_seed(0)
    g = torch.Generator().manual_seed(0)
    if mode == "head":
        B, H, W = 8, 288, 1280
        model = RetinanetHead(**cfg.head).cuda().train()
        head = model
        feats = [torch.randn(B, 256, (H + 2 ** l - 1) // 2 ** l, (W + 2 ** l - 1) // 2 ** l, generator=g).cuda() for l in range(3, 8)]
        ann = torch.from_numpy(odd_rows(fx["train/ann"])).cuda()
    else:
        B, H, W = 2, 96, 320
        model = RetinaNet(cfg).cuda().train()
        head = model.bbox_head
        img = torch.randn(B, 3, H, W, generator=g).cuda()
        ann = torch.from_numpy(odd_rows(fx["argmax/ann"])).cuda()
    with torch.no_grad():                       # retina_cls / retina_reg start at zero weights (retinanet_head.py:64-69): give them values
        for seq in (head.retina_cls, head.retina_reg):
            seq[0].weight.copy_(torch.randn(seq[0].weight.shape, generator=g) * 1e-2)
            seq[0].bias.add_((torch.randn(seq[0].bias.shape, generator=g) * 0.5).cuda())

    def step():
        torch.manual_seed(0)
        model.zero_grad()
        if mode == "head":
            cls, reg = head(feats)
            c, r, d = head.loss(cls, reg, head.get_anchor(torch.zeros(B, 3, H, W, device="cuda")), ann)
        else:
            c, r, d = model([img, ann, None])
        (c + r).backward()
        torch.cuda.synchronize()
        return c.item(), float(r), d["total_loss"].item(), {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}

    ref = step()
    plugin.install_retinanet_loss_into_reference()
    native_bound = RetinanetHead.loss is retina_loss.head_loss
    nat = step()
    rel = lambda a, b: abs(a - b) / max(abs(b), 1e-30)  # noqa: E731
    # A conv bias ahead of a train-mode BatchNorm has an analytically zero gradient: what both runs hold there is rounding noise, so
    # those tensors (reference max |grad| below 1e-6 of the largest gradient) are held to that noise floor, the rest to their max.
    top = max(float(gr.abs().max()) for gr in ref[3].values())
    noise = {n for n, gr in ref[3].items() if float(gr.abs().max()) <= 1e-6 * top}
    grad_err = {n: float((nat[3][n] - gr).abs().max() / (top if n in noise else gr.abs().max())) for n, gr in ref[3].items()}
    out = dict(mode=mode, native_bound=native_bound, cls=[nat[0], ref[0]], reg=[nat[1], ref[1]], cls_rel=rel(nat[0], ref[0]),
               reg_rel=rel(nat[1], ref[1]), total_rel=rel(nat[2], ref[2]), n_grads=len(grad_err), same_params=sorted(nat[3]) == sorted(ref[3]),
               grad_err_max=max(grad_err.values()), grad_err_worst=max(grad_err, key=grad_err.get), noise_floor_tensors=sorted(noise))
    print("SEAM_JSON " + json.dumps(out))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "head")
