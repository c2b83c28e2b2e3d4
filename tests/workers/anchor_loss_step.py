"""Worker of tests/test_anchor_loss_gpu.py::test_reference_head_training_step (own process, GPU box).

One training step of the reference's UNMODIFIED StereoHead (Stereo3D_example head: 1408-channel features, 2 classes) on the GPU at
Stereo3D's training shape (B=4, 288x1280), first with its own Python loss, then with `plugin.install_loss_into_reference()` in place:
the same features, dropout masks and annotations.  Prints one JSON line with the loss and head-parameter gradient differences."""
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import refload  # noqa: E402


def main():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False
    from visualdet3d_b200.ops import dcn as our_dcn, iou3d as our_iou
    from visualdet3d_b200 import anchor_loss, plugin, synth
    refload.load_reference(device="cuda", dcn_ext=our_dcn, iou3d_ext=our_iou)
    from visualDet3D.networks.heads.detection_3d_head import StereoHead

    obj_types = ["Car", "Pedestrian"]
    tmp = tempfile.mkdtemp()
    pm, ps = synth.synth_priors(16, 3, obj_types)
    synth.write_priors(tmp, pm, ps, obj_types)
    hc = synth.stereo3d_cfg(tmp, obj_types).head
    head = StereoHead(**refload.to_edict(dict(hc))).cuda().train()
    g = torch.Generator().manual_seed(0)
    with torch.no_grad():                       # the output convs start at zero (detection_3d_head.py:520-533): give them values
        for seq in (head.cls_feature_extraction, head.reg_feature_extraction):
            seq[-2].weight.copy_(torch.randn(seq[-2].weight.shape, generator=g) * 1e-3)
            seq[-2].bias.copy_(torch.randn(seq[-2].bias.shape, generator=g) * 0.5)
    B, H, W = 4, 288, 1280
    feats = (torch.randn(B, hc.layer_cfg.num_features_in, H // 16, W // 16, generator=g)).cuda()
    P2 = synth.synth_P2(B, H, W)[0].cuda()
    anchors = head.get_anchor(torch.zeros(B, 3, H, W, device="cuda"), P2)
    fx = np.load(os.path.join(ROOT, "tests", "golden", "anchor_loss.npz"))
    ann = torch.from_numpy(fx["a/ann"]).cuda()

    def step():
        torch.manual_seed(0)
        head.zero_grad()
        cls, reg = head({"features": feats})
        c, r, d = head.loss(cls, reg, anchors, ann, P2)
        (c + r).sum().backward()
        torch.cuda.synchronize()
        return c.item(), r.item(), d["total_loss"].item(), {n: p.grad.clone() for n, p in head.named_parameters() if p.grad is not None}

    ref = step()
    plugin.install_loss_into_reference()
    native_bound = StereoHead.loss is anchor_loss.head_loss
    nat = step()
    rel = lambda a, b: abs(a - b) / max(abs(b), 1e-30)  # noqa: E731
    # A conv bias ahead of a train-mode BatchNorm has an analytically zero gradient: what both runs hold there is rounding noise, so
    # those tensors (reference max |grad| below 1e-6 of the largest head gradient) are held to that noise floor, the rest to their max.
    top = max(float(gr.abs().max()) for gr in ref[3].values())
    noise = {n for n, gr in ref[3].items() if float(gr.abs().max()) <= 1e-6 * top}
    grad_err = {n: float((nat[3][n] - gr).abs().max() / (top if n in noise else gr.abs().max())) for n, gr in ref[3].items()}
    out = dict(native_bound=native_bound, cls=[nat[0], ref[0]], reg=[nat[1], ref[1]], cls_rel=rel(nat[0], ref[0]),
               reg_rel=rel(nat[1], ref[1]), total_rel=rel(nat[2], ref[2]), n_grads=len(grad_err), same_params=sorted(nat[3]) == sorted(ref[3]),
               grad_err_max=max(grad_err.values()), grad_err_worst=max(grad_err, key=grad_err.get), noise_floor_tensors=sorted(noise))
    print("SEAM_JSON " + json.dumps(out))


if __name__ == "__main__":
    main()
