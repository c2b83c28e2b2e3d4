"""Worker of tests/test_km3d_loss_gpu.py::test_reference_head_training_step (own process, GPU box).

One training step of the reference's UNMODIFIED KM3DHead (KM3D_example head layers: 64-channel features, 256-channel head convs, 3
classes) on the GPU at B = 8 on 96x320 maps, first with its own Python loss -- boxes_iou3d_gpu running the reference's own compiled iou3d
extension (oracle/_ref ref_iou3d_cuda) -- then with `plugin.install_km3d_loss_into_reference()` in place, which reads meta['P2'],
meta['epoch'] and the head's position_loss.output_w and rampup_length.  Targets are those of tests/golden/km3d_loss.npz case a, at epoch 37.
The head's output convs start near zero and their outputs are added to the fixture's head outputs, so the solved positions land near the
targets and the box scores lie inside (0, 1) as in training (with freshly initialised output convs every keypoint would sit on its pixel).
The annotations are rebuilt for each arm: the reference rewrites annotations['dep'] in place.  The reference step runs twice, with two
draws of its randn * 1e-8 jitter of A^T A: the difference between those two is the reference's own scatter.
Prints one JSON line with the loss and head-parameter gradient differences, native against the first reference run and the second
reference run against the first."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402
import build_ref  # noqa: E402
import refload  # noqa: E402


def main():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False
    from visualdet3d_b200.ops import dcn as our_dcn
    from visualdet3d_b200 import km3d_loss, plugin
    from visualdet3d_b200.detectors import km3d_cfg
    from conftest import load_fixture
    ref_iou3d = build_ref.load("ref_iou3d_cuda")
    refload.load_reference(device="cuda", dcn_ext=our_dcn, iou3d_ext=ref_iou3d)
    from visualDet3D.networks.heads.km3d_head import KM3DHead
    from visualDet3D.networks.lib.ops.iou3d import iou3d as ref_iou3d_py
    import importlib.util
    spec = importlib.util.spec_from_file_location("gen", os.path.join(ROOT, "tests", "golden", "make_golden_km3d_loss.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)

    fx = load_fixture("km3d_loss")["a"]
    hc = km3d_cfg().head
    head = KM3DHead(**refload.to_edict(dict(hc))).cuda().train()
    assert head.position_loss.output_w == int(fx["W"]) and head.rampup_length == gen.RAMPUP
    g = torch.Generator().manual_seed(0)
    with torch.no_grad():                       # small output convs: the maps stay near the fixture's
        for name, seq in head.head_layers.items():
            seq[-1].weight.copy_(torch.randn(seq[-1].weight.shape, generator=g) * 0.002)
            seq[-1].bias.copy_(torch.randn(seq[-1].bias.shape, generator=g) * 0.01)
    B, H, W = int(fx["B"]), int(fx["H"]), int(fx["W"])
    feats = torch.randn(B, hc.layer_cfg.input_features, H, W, generator=g).cuda()
    base = {k: v.cuda() for k, v in gen.head_outputs(fx).items()}
    P2 = torch.from_numpy(fx["P2"]).cuda()

    def step(seed=0):
        torch.manual_seed(seed)                 # the reference's randn jitter of A^T A in gen_position
        head.zero_grad()
        ann = {k: v.cuda() for k, v in gen.annotations(fx).items()}
        out = {k: v + base[k] for k, v in head(feats).items()}
        loss, stats = head.loss(out, ann, dict(P2=P2, epoch=gen.GRAD_EPOCH))
        loss.backward()
        torch.cuda.synchronize()
        return {k: float(v) for k, v in stats.items()}, {n: p.grad.clone() for n, p in head.named_parameters() if p.grad is not None}

    ref = step()
    ref1 = step(1)                              # the reference's own scatter: the same step with another jitter draw
    ref_kernel = ref_iou3d_py.boxes_overlap_bev_gpu is ref_iou3d.boxes_overlap_bev_gpu
    plugin.install_km3d_loss_into_reference()
    native_bound = KM3DHead.loss is km3d_loss.head_loss
    nat = step()
    lrel = lambda x, y: {k: abs(x[0][k] - v) / max(abs(v), 1e-30) for k, v in y[0].items()}  # noqa: E731
    gerr = lambda x, y: {n: float((x[1][n] - gr).abs().max() / gr.abs().max().clamp_min(1e-30)) for n, gr in y[1].items()}  # noqa: E731
    rel, grad_err = lrel(nat, ref), gerr(nat, ref)
    ref_rel, ref_grad = lrel(ref1, ref), gerr(ref1, ref)
    out = dict(native_bound=native_bound, reference_iou3d_kernel=ref_kernel, loss=[nat[0]["total_loss"], ref[0]["total_loss"]],
               box_score=[nat[0]["box_score"], ref[0]["box_score"]], loss_rel=rel, n_grads=len(grad_err),
               same_params=sorted(nat[1]) == sorted(ref[1]), grad_err=grad_err, ref_scatter_loss=ref_rel, ref_scatter_grad=ref_grad)
    print("SEAM_JSON " + json.dumps(out))


if __name__ == "__main__":
    main()
