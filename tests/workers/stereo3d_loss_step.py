"""Worker of tests/test_disparity_loss_gpu.py::test_reference_stereo3d_training_step (own process, GPU box).

One training step of the reference's UNMODIFIED Stereo3D (Stereo3D_example, pretrained=False, seeded synthetic weights) in train mode on
the GPU at its training shape (B=4, 288x1280): `train_forward` + backward, first with the reference's own anchor-head and disparity losses,
then with `plugin.install_loss_into_reference()` and `plugin.install_disparity_loss_into_reference()` in place.  The annotations are
tests/golden/anchor_loss.npz case a, the disparity label tests/golden/disparity_loss.npz case a (regenerated from its seed).  Deterministic
cuDNN, no TF32, the same seed before each step.  Prints one JSON line with the loss differences and, per parameter group (the depth_output
branch, fed by the disparity loss only; the bbox_head, fed by the anchor loss only; the shared trunk), the largest gradient difference
over each tensor's max |.|."""
import importlib.util
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


def golden_module():
    path = os.path.join(ROOT, "tests", "golden", "make_golden_disparity_loss.py")
    spec = importlib.util.spec_from_file_location("make_golden_disparity_loss", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def group(name: str) -> str:
    if ".depth_output." in name:
        return "depth"
    if name.startswith("bbox_head."):
        return "head"
    return "trunk"


def main():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False
    from visualdet3d_b200.ops import dcn as our_dcn, iou3d as our_iou
    from visualdet3d_b200 import disparity_loss, plugin, synth
    refload.load_reference(device="cuda", dcn_ext=our_dcn, iou3d_ext=our_iou)
    from visualDet3D.networks.utils import registry as ref_registry
    from visualDet3D.networks.heads import losses as ref_losses

    obj = ["Car", "Pedestrian"]
    tmp = tempfile.mkdtemp()
    pm, ps = synth.synth_priors(16, 3, obj)
    synth.write_priors(tmp, pm, ps, obj)
    cfg = refload.to_edict(dict(obj_types=obj, detector=synth.stereo3d_cfg(tmp, obj)))
    det = ref_registry.DETECTOR_DICT["Stereo3D"](cfg.detector)
    det.load_state_dict(synth.synth_state_dict({k: tuple(v.shape) for k, v in det.state_dict().items()}, 0), strict=False)
    det = det.cuda().train()
    B, H, W = 4, 288, 1280
    left, right, P2, P3 = (t.cuda() for t in synth.synth_stereo_inputs(B, H, W, seed=1))
    P2 = synth.synth_P2(B, H, W)[0].cuda()              # the P2 the anchor fixture's annotations were drawn for
    ann = torch.from_numpy(np.load(os.path.join(ROOT, "tests", "golden", "anchor_loss.npz"))["a/ann"]).cuda()
    _, disp = golden_module().inputs("a")
    disp = disp.cuda()

    def step():
        torch.manual_seed(0)
        det.zero_grad()
        cls, reg, d = det.train_forward(left, right, ann, P2, P3, disp)
        (cls + reg).mean().backward()
        torch.cuda.synchronize()
        grads = {n: p.grad.clone() for n, p in det.named_parameters() if p.grad is not None}
        return float(cls.mean()), float(reg.mean()), float(d["disparity_loss"]), grads

    ref = step()
    plugin.install_loss_into_reference()
    plugin.install_disparity_loss_into_reference()
    native_bound = ref_losses.DisparityLoss.forward is disparity_loss.forward
    nat = step()
    rel = lambda a, b: abs(a - b) / max(abs(b), 1e-30)  # noqa: E731
    out = dict(native_bound=native_bound, cls=[nat[0], ref[0]], reg=[nat[1], ref[1]], disp=[nat[2], ref[2]], cls_rel=rel(nat[0], ref[0]),
               reg_rel=rel(nat[1], ref[1]), disp_rel=rel(nat[2], ref[2]), disp_loss_ran=ref[2] != 0.0,
               same_params=sorted(nat[3]) == sorted(ref[3]))
    # A conv bias ahead of a train-mode BatchNorm has an analytically zero gradient: what both runs hold there is rounding noise, so those
    # tensors (max |grad| below 1e-6 of their group's largest) are held to the group's largest, the rest to their own max.
    for grp in ("depth", "head", "trunk"):
        names = [n for n in ref[3] if group(n) == grp]
        top = max(float(ref[3][n].abs().max()) for n in names)
        err = {}
        for n in names:
            m = float(ref[3][n].abs().max())
            err[n] = float((nat[3][n] - ref[3][n]).abs().max()) / (top if m <= 1e-6 * top else m)
        worst = max(err, key=err.get)
        out[f"{grp}_grad_err"], out[f"{grp}_grad_worst"], out[f"{grp}_tensors"] = err[worst], worst, len(names)
    print("SEAM_JSON " + json.dumps(out))


if __name__ == "__main__":
    main()
