"""-m gpu: Yolo3D (DCNv2 head) and GroundAwareYolo3D (LookGround head) against the reference fixtures and the CPU oracle."""
import numpy as np
import pytest
import torch

from conftest import load_fixture, subsample_like
import torch_port as tp
from detector_harness import assert_dets_match, run_with_stages

pytestmark = pytest.mark.gpu


def build(kind):
    from visualdet3d_b200.detectors import build_synthetic_mono3d
    det, sd, cfg, priors = build_synthetic_mono3d(kind, seed=0)
    return det.cuda().eval(), sd, cfg, priors


@pytest.mark.parametrize("kind,tag", [("Yolo3D", "yolo3d_96x320"), ("Yolo3D", "yolo3d_288x1280"),
                                      ("GroundAwareYolo3D", "groundawareyolo3d_96x320"), ("GroundAwareYolo3D", "groundawareyolo3d_288x640"),
                                      ("GroundAwareYolo3D", "groundawareyolo3d_288x1280")])     # the last one = BASELINE configs[2] shape
def test_against_reference_fixture(kind, tag):
    from visualdet3d_b200 import synth
    det, sd, cfg, (pm, ps) = build(kind)
    fx = load_fixture(tag)
    H, W, B, seed = [int(v) for v in fx["meta"]]
    img, P2 = synth.synth_mono_inputs(B, H, W, seed=1)
    res, st = run_with_stages(det, img, P2, flatten_heads=True)
    rep = {nm: float(np.abs(subsample_like(st[nm], fx[nm]) - fx[nm]["samples"]).max())
           for nm in ["features", "cls_preds", "reg_preds"] + (["gac"] if "gac" in fx else [])}
    print(tag, "stage max|diff| vs reference:", rep)
    assert all(v < 5e-4 for v in rep.values()), rep
    ref = tp.mono3d_forward(sd, img, P2, cfg, pm, ps)
    for b in range(B):
        np.testing.assert_array_equal(np.packbits(st["mask"][b].numpy().astype(bool)), fx[f"mask_{b}"])
        k = len(res[b][0])
        assert k == len(fx[f"scores_{b}"])
        swaps = assert_dets_match(res[b], ref[b], det._last_decoder.anchor[b, :k])
        if swaps == 0:
            np.testing.assert_allclose(res[b][0].cpu().numpy(), fx[f"scores_{b}"], atol=1e-3)
            np.testing.assert_allclose(res[b][1].cpu().numpy(), fx[f"bboxes_{b}"], atol=1e-3)
            np.testing.assert_array_equal(res[b][2].cpu().numpy(), fx[f"cls_{b}"])


def test_look_ground_op_vs_oracle():
    """LookGround in isolation (R/lib/look_ground.py:24-71) incl. per-image P2 and rows sampled past the bottom border."""
    from visualdet3d_b200 import engine as E, synth
    from visualdet3d_b200.detectors import modules as M
    from visualdet3d_b200.detectors.mono3d import LookGroundRunner
    g = torch.Generator().manual_seed(0)
    C, B, H, W = 64, 3, 18, 80
    m = M.LookGroundP(C)
    m.disp_create[0].weight.data = torch.randn(1, C, 3, 3, generator=g) * 0.05
    m.disp_create[0].bias.data = torch.randn(1, generator=g)
    m.extract.weight.data = torch.randn(C, C + 1, 1, 1, generator=g) * 0.1
    m.extract.bias.data = torch.randn(C, generator=g) * 0.1
    m.alpha.data = torch.tensor([0.7])
    sd = {"g." + k: v.detach().clone() for k, v in m.state_dict().items()}
    x = torch.randn(B, C, H, W, generator=g)
    _, P2 = synth.synth_mono_inputs(B, 16 * H, 16 * W, seed=3)
    ref = tp.look_ground(sd, "g", x, P2)
    run = LookGroundRunner(m, "cuda")
    ar = E.Arena()
    comp = torch.zeros(2, B, H, W, C, device="cuda", dtype=torch.float16) if ar.lo_form == "h16" else torch.zeros(B, H, W, C, device="cuda")
    xa = E.split_lo(E.Act(x.permute(0, 2, 3, 1).contiguous().cuda(), 0, None, comp))
    out = run.run(xa, P2.cuda(), ar)
    np.testing.assert_allclose(out.to_nchw().cpu().numpy(), ref.numpy(), rtol=1e-4, atol=2e-5)


def test_batch8_288x1280_gac_all_images_vs_oracle():
    """BASELINE configs[2] shape (GAC head, batch 8 mono 288x1280): determinism, batch invariance, and EVERY image vs the oracle."""
    from visualdet3d_b200 import synth
    det, sd, cfg, (pm, ps) = build("GroundAwareYolo3D")
    img, P2 = synth.synth_mono_inputs(8, 288, 1280, seed=5)
    ic, pc = img.cuda(), P2.cuda()
    with torch.no_grad():
        r1 = det.forward_batch(ic, pc)
        anchors = [det._last_decoder.anchor[b, :len(r1[b][0])].clone() for b in range(8)]
        r2 = det.forward_batch(ic, pc)
        single = det([ic[3:4], pc[3:4]])
    assert all(torch.equal(x, y) for a, b in zip(r1, r2) for x, y in zip(a, b))
    assert all(torch.equal(x, y) for x, y in zip(r1[3], single))
    ref = tp.mono3d_forward(sd, img, P2, cfg, pm, ps)
    swaps = [assert_dets_match(r1[b], ref[b], anchors[b]) for b in range(8)]
    print("GAC 8 x 288x1280: detections per image", [len(r[0]) for r in r1], "score-tied order swaps", swaps)
