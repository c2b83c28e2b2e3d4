"""Worker of tests/test_monoflex_loss_gpu.py::test_reference_head_training_step (own process, GPU box).

One training step of the reference's UNMODIFIED MonoFlexHead (Monoflex_example head layers: 64-channel features, 256-channel head
convs, 3 classes) on the GPU at B = 8 on 96x320 maps, first with its own Python loss, then with
`plugin.install_monoflex_loss_into_reference()` in place: the same features and the targets of tests/golden/monoflex_loss.npz case a.
Prints one JSON line with the loss and head-parameter gradient differences."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402
import refload  # noqa: E402


def main():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False
    from visualdet3d_b200.ops import dcn as our_dcn, iou3d as our_iou
    from visualdet3d_b200 import monoflex_loss, plugin
    from visualdet3d_b200.detectors import monoflex_cfg
    from conftest import load_fixture
    refload.load_reference(device="cuda", dcn_ext=our_dcn, iou3d_ext=our_iou)
    from visualDet3D.networks.heads.monoflex_head import MonoFlexHead
    import importlib.util
    spec = importlib.util.spec_from_file_location("gen", os.path.join(ROOT, "tests", "golden", "make_golden_monoflex_loss.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)

    fx = load_fixture("monoflex_loss")["a"]
    hc = monoflex_cfg().head
    head = MonoFlexHead(**refload.to_edict(dict(hc))).cuda().train()
    g = torch.Generator().manual_seed(0)
    with torch.no_grad():                       # the output convs start at (near) zero: give them values
        for name, seq in head.head_layers.items():
            seq[-1].weight.copy_(torch.randn(seq[-1].weight.shape, generator=g) * 0.02)
            seq[-1].bias.copy_(torch.randn(seq[-1].bias.shape, generator=g) * 0.5 + (-2.19 if name == "hm" else 0.0))
    B, H, W = int(fx["B"]), int(fx["H"]), int(fx["W"])
    feats = torch.randn(B, hc.layer_cfg.input_features, H, W, generator=g).cuda()
    P2 = torch.from_numpy(fx["P2"]).cuda()

    def step():
        head.zero_grad()
        ann = {k: v.cuda() for k, v in gen.annotations(fx).items()}
        out = head(feats)
        # the reference's _gather_output indexes a host arange with the device reg_mask, which torch refuses since 2.x: under a cuda
        # default device the arange is made on the device (no source edit)
        with torch.device("cuda"):
            loss, stats = head.loss(out, ann, dict(P2=P2, epoch=0))
        loss.mean().backward()
        torch.cuda.synchronize()
        return {k: float(v) for k, v in stats.items()}, {n: p.grad.clone() for n, p in head.named_parameters() if p.grad is not None}

    ref = step()
    plugin.install_monoflex_loss_into_reference()
    native_bound = MonoFlexHead.loss is monoflex_loss.head_loss
    nat = step()
    rel = {k: abs(nat[0][k] - v) / max(abs(v), 1e-30) for k, v in ref[0].items()}
    grad_err = {n: float((nat[1][n] - gr).abs().max() / gr.abs().max().clamp_min(1e-30)) for n, gr in ref[1].items()}
    out = dict(native_bound=native_bound, loss=[nat[0]["total_loss"], ref[0]["total_loss"]], loss_rel=rel, loss_rel_max=max(rel.values()),
               n_grads=len(grad_err), same_params=sorted(nat[1]) == sorted(ref[1]), grad_err_max=max(grad_err.values()),
               grad_err_worst=max(grad_err, key=grad_err.get))
    print("SEAM_JSON " + json.dumps(out))


if __name__ == "__main__":
    main()
