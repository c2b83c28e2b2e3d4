"""-m gpu: the sub-pixel phase transposed conv (vd3d_convtranspose2d_tc16) alone, and KM3D_example / MonoFlex on the ResNet-18 CenterNet
core against the reference fixtures (tests/golden/make_golden_km3d_resnet.py) and the CPU oracle."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN, load_fixture, subsample_like
import centernet_resnet_oracle as ro
from detector_harness import match_dets, run_with_stages

pytestmark = pytest.mark.gpu


def _planes_act(x_nchw):
    """NCHW fp32 -> an engine activation with fresh fp16 (hi, lo) planes"""
    from visualdet3d_b200 import engine as E
    t = x_nchw.permute(0, 2, 3, 1).contiguous().cuda()
    a = E.Act(t, 0, None, torch.zeros((2,) + tuple(t.shape), dtype=torch.float16, device="cuda"))
    return E.split_lo(a)


@pytest.mark.parametrize("Cin", [512, 256])
@pytest.mark.parametrize("B,H,W", [(1, 1, 1), (2, 3, 5), (3, 7, 13), (1, 12, 40), (2, 48, 160)])
def test_transposed_conv_layer(Cin, B, H, W):
    """vs F.conv_transpose2d in float64 with the BatchNorm folded and ReLU: every tile edge (16 x 8 tiles over the input grid) and both
    borders of every phase; the fp32 output and the planes-only output, and the planes equal the fp16 split of the fp32 tensor."""
    from visualdet3d_b200 import engine as E
    Cout = 256
    g = torch.Generator().manual_seed(Cin + 7 * B + 31 * H + W)
    wt = torch.randn(Cin, Cout, 4, 4, generator=g) * (2.0 / (4 * Cin)) ** 0.5
    bn = dict(weight=torch.rand(Cout, generator=g) + 0.5, bias=torch.randn(Cout, generator=g) * 0.1,
              running_mean=torch.randn(Cout, generator=g) * 0.1, running_var=torch.rand(Cout, generator=g) + 0.5)
    x = torch.randn(B, Cin, H, W, generator=g)
    ref = F.relu(F.batch_norm(F.conv_transpose2d(x.double(), wt.double(), None, stride=2, padding=1), bn["running_mean"].double(),
                              bn["running_var"].double(), bn["weight"].double(), bn["bias"].double(), training=False, eps=1e-5))
    layer = E.ConvTransposeLayer(wt, bn, relu=True, device="cuda")
    xa = _planes_act(x)
    out = E.Act(torch.full((B, 2 * H, 2 * W, Cout), float("nan"), device="cuda"), 0, None,
                torch.full((2, B, 2 * H, 2 * W, Cout), float("nan"), dtype=torch.float16, device="cuda"))
    layer(xa, out)
    torch.cuda.synchronize()
    got = out.t.permute(0, 3, 1, 2).double().cpu()
    scale = max(1.0, float(ref.abs().max()))
    err = float((got - ref).abs().max())
    print(f"Cin {Cin} B {B} {H}x{W}: max|diff| {err:.2e} (max|ref| {scale:.2f})")
    assert err < 1e-5 * scale, err
    hi = out.t.half()
    assert torch.equal(out.lo[0], hi) and torch.equal(out.lo[1], (out.t - hi.float()).half())
    # planes-only output: the same values, no fp32 copy written
    out2 = E.Act(torch.full((B, 2 * H, 2 * W, Cout), float("nan"), device="cuda"), 0, None,
                 torch.zeros((2, B, 2 * H, 2 * W, Cout), dtype=torch.float16, device="cuda"))
    layer(xa, out2, f32_out=False)
    torch.cuda.synchronize()
    assert not out2.f32 and bool(torch.isnan(out2.t).all())
    assert torch.equal(out2.lo, out.lo)


@pytest.fixture(scope="module")
def km3d():
    from visualdet3d_b200.detectors import build_synthetic_monoflex
    det, sd, cfg = build_synthetic_monoflex(seed=0, name="KM3D", backbone="resnet18")
    return det.cuda().eval(), sd, cfg


@pytest.mark.parametrize("tag", ["km3d_resnet_96x320", "km3d_resnet_192x640", "km3d_resnet_384x1280"])
def test_km3d_example_against_reference_fixture_and_oracle(km3d, tag):
    """KM3D_example (ResNet-18 + transposed-conv up-sampling): features and head maps within 1e-3 of the reference, kept peak sets identical,
    detections within 1e-3 of the oracle except cx / cy / z, which must lie within 1e-3 + the reference's own spread of its envelope
    (gen_position's randn jitter, tests/golden/km3d_resnet_spread.npz)."""
    from visualdet3d_b200 import synth
    det, sd, cfg = km3d
    fx = load_fixture(tag)
    H, W, B, seed = [int(v) for v in fx["meta"]]
    img, P2 = synth.synth_mono_inputs(B, H, W, seed=1)
    res, st = run_with_stages(det, img, P2)
    rep = {"features": float(np.abs(subsample_like(st["features"], fx["features"]) - fx["features"]["samples"]).max())}
    off = det._plan["offsets"]
    for n, k in cfg["head"]["layer_cfg"]["head_dict"].items():
        rep[n] = float(np.abs(subsample_like(st["heads"][:, off[n]:off[n] + k], fx["head_" + n]) - fx["head_" + n]["samples"]).max())
    print(tag, "stage max|diff| vs reference:", rep)
    assert all(v < 1e-3 for v in rep.values()), rep
    ref = ro.km3d_forward(sd, img, P2, cfg)
    env = np.load(os.path.join(GOLDEN, "km3d_resnet_spread.npz"))
    for b in range(B):
        k = len(res[b][0])
        assert k == len(fx[f"scores_{b}"]) and k > 3
        gi = det._last_decoder.anchor[b, :k].cpu().long()
        rs, rb, rc, rflat = ref[b]
        assert torch.equal(torch.sort(gi)[0], torch.sort(rflat)[0]), "kept peak sets differ"
        pos = {int(a): i for i, a in enumerate(rflat.tolist())}
        perm = torch.tensor([pos[int(a)] for a in gi.tolist()])
        s, bx, ci = [t.cpu() for t in res[b]]
        for i in (perm != torch.arange(k)).nonzero()[:, 0].tolist():
            assert abs(float(rs[perm[i]]) - float(rs[i])) < 1e-5, "order differs between rows that are not score-tied"
        assert torch.equal(ci.view(-1), rc[perm].view(-1))
        assert float((s - rs[perm]).abs().max()) < 1e-3
        d = (bx - rb[perm]).abs().numpy()
        lo, hi = env[f"{H}x{W}_{b}/min"][perm.numpy()], env[f"{H}x{W}_{b}/max"][perm.numpy()]
        out_of_env = np.maximum(lo - bx.numpy(), bx.numpy() - hi).clip(min=0)
        spread = (hi.astype(np.float64) - lo).astype(np.float32)
        print(tag, b, "max |diff| vs oracle per column", np.array2string(d.max(0), precision=2),
              "| distance to the reference envelope", np.array2string(out_of_env.max(0), precision=2))
        other = [0, 1, 2, 3, 7, 8, 9, 10]
        assert float(d[:, other].max()) < 1e-3, d[:, other].max(0)
        assert bool((out_of_env[:, 4:7] <= 1e-3 + spread[:, 4:7]).all()), (out_of_env[:, 4:7] - spread[:, 4:7]).max(0)


def test_monoflex_resnet_against_reference_fixture():
    from visualdet3d_b200 import synth
    from visualdet3d_b200.detectors import build_synthetic_monoflex
    det, sd, cfg = build_synthetic_monoflex(seed=0, name="MonoFlex", backbone="resnet18")
    det = det.cuda().eval()
    fx = load_fixture("monoflex_resnet_96x320")
    H, W, B, seed = [int(v) for v in fx["meta"]]
    img, P2 = synth.synth_mono_inputs(B, H, W, seed=1)
    res, st = run_with_stages(det, img, P2)
    rep = {"features": float(np.abs(subsample_like(st["features"], fx["features"]) - fx["features"]["samples"]).max())}
    off = det._plan["offsets"]
    for n, k in cfg["head"]["layer_cfg"]["head_dict"].items():
        rep[n] = float(np.abs(subsample_like(st["heads"][:, off[n]:off[n] + k], fx["head_" + n]) - fx["head_" + n]["samples"]).max())
    print("MonoFlex-ResNet stage max|diff| vs reference:", rep)
    assert all(v < 1e-3 for v in rep.values()), rep
    ref = ro.monoflex_forward(sd, img, P2, cfg)
    for b in range(B):
        k = len(res[b][0])
        assert k == len(fx[f"scores_{b}"]) and k > 3
        match_dets(res[b], ref[b], det._last_decoder.anchor[b, :k])
        if torch.equal(det._last_decoder.anchor[b, :k].cpu().long(), ref[b][3]):
            np.testing.assert_allclose(res[b][0].cpu().numpy(), fx[f"scores_{b}"], atol=1e-3, rtol=0)
            np.testing.assert_allclose(res[b][1].cpu().numpy(), fx[f"bboxes_{b}"], atol=1e-3, rtol=1e-5)
            np.testing.assert_array_equal(res[b][2].cpu().numpy().reshape(-1), fx[f"cls_{b}"].reshape(-1))


def test_batch8_384x1280_determinism_batch_invariance_graphs_and_planes(km3d, monkeypatch):
    """KM3D_example at batch 8, 384x1280: two runs identical, image b of the batch bit-identical to the single-image call, CUDA-graph replay
    equal to eager launches, and (engine.CHECK_LO) fresh fp16 planes in front of every tensor-core conv."""
    from visualdet3d_b200 import engine, graphs, synth
    det = km3d[0]
    img, P2 = synth.synth_mono_inputs(8, 384, 1280, seed=9)
    ic, pc = img.cuda(), P2.cuda()
    with torch.no_grad():
        r1 = det.forward_batch(ic, pc)
        r2 = det.forward_batch(ic, pc)
        single = det([ic[5:6], pc[5:6]])
    assert all(torch.equal(x, y) for a, b in zip(r1, r2) for x, y in zip(a, b))
    assert all(torch.equal(x, y) for x, y in zip(r1[5], single))
    assert all(len(r[0]) > 3 for r in r1)
    print("KM3D-ResNet 8 x 384x1280: detections per image", [len(r[0]) for r in r1])
    kmax = 128
    rec = torch.zeros(8, 1 + kmax * 13, device="cuda")
    step = graphs.GraphedStep(det, [ic], pc, rec, kmax)
    with torch.no_grad():
        step()
        eager = rec.clone()
        step()
        step()
    torch.cuda.synchronize()
    assert step.graph is not None and step.replays >= 1
    assert torch.equal(rec, eager)
    for b in range(8):
        assert int(eager[b, 0]) == len(r1[b][0])
    monkeypatch.setattr(engine, "CHECK_LO", True)
    with torch.no_grad():
        r3 = det.forward_batch(ic, pc)
    assert all(torch.equal(x, y) for a, b in zip(r1, r3) for x, y in zip(a, b))
