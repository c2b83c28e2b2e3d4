"""-m gpu: the RetinaNet 2-D detector against the reference fixtures (tests/golden/make_golden_retinanet.py), its device decode on the
reference's own head outputs, the fused FPN top-down add, batch invariance and CUDA-graph replay."""
import numpy as np
import pytest
import torch

from conftest import load_fixture, subsample_like
from detector_harness import run_with_stages

pytestmark = pytest.mark.gpu


def build(nms_pre=1000):
    from visualdet3d_b200.detectors import build_synthetic_retinanet
    det, sd, cfg = build_synthetic_retinanet(seed=0, nms_pre=nms_pre)
    return det.cuda().eval(), sd, cfg


def test_decode_stage_on_reference_head_outputs():
    """top-k order, NMS keep set, labels, scores and boxes from the reference's own cls / reg tensors."""
    from visualdet3d_b200.detectors.retinanet import RetinaDecode
    det, _, cfg = build()
    fx = load_fixture("retinanet_96x320")
    B = int(fx["meta"][2])
    cls = torch.tensor(fx["cls_full"]).cuda().contiguous()           # [B, N, C]
    reg = torch.tensor(fx["reg_full"]).cuda().contiguous()           # [B, N, 4]
    anchors = torch.tensor(fx["anchors_full"]).cuda().contiguous()
    N, C, A = cls.shape[1], cls.shape[2], det.num_anchors
    tc = cfg.head.test_cfg
    dec = RetinaDecode(B, N, tc.nms_pre, "cuda")

    def run(score_thr, iou_thr):
        # one "level" of N / A pixels with channel pitch A * C (A * 4): element (n, c) at n * C + c, the layout of the reference's tensors
        dec.run_levels([cls], [reg], [N // A], A * C, A * 4, anchors, A, C, tc.nms_pre, [0.0] * 4, [1.0] * 4, score_thr, iou_thr)
        return [(s.cpu(), b[:, :4].cpu(), c.cpu(), dec.anchor[i, :len(s)].cpu().long()) for i, (s, b, c) in enumerate(dec.results())]

    # no suppression (IoU > 1 never holds) and no threshold: the k candidates in the top-k order
    for b, (s, _, _, idx) in enumerate(run(0.0, 1.0)):
        np.testing.assert_array_equal(idx.numpy(), fx[f"topk_{b}"])
    # the reference's NMS keep set above score_thr (the generator asserts IoU margins among exactly these candidates)
    out = run(tc.score_thr, tc.nms_iou_thr)
    for b in range(B):
        s, bx, c, idx = out[b]
        assert len(s) == len(fx[f"scores_{b}"]) > 0
        np.testing.assert_array_equal(idx.numpy(), fx[f"topk_{b}"][fx[f"keep_{b}"]][:len(s)])
        np.testing.assert_array_equal(c.numpy(), fx[f"cls_{b}"])
        print("decode stage: max |dscore|", float(np.abs(s.numpy() - fx[f"scores_{b}"]).max()),
              "max |dbox|", float(np.abs(bx.numpy() - fx[f"bboxes_{b}"]).max()), "max |box|", float(np.abs(fx[f"bboxes_{b}"]).max()))
        np.testing.assert_allclose(s.numpy(), fx[f"scores_{b}"], rtol=0, atol=1e-6)
        # boxes: the same expression order as the reference; the device expf may differ from the host's by an ulp, which at coordinates of
        # hundreds of pixels is ~3e-5 absolute, so the bound is in ulps (measured: at most 1)
        np.testing.assert_array_max_ulp(bx.numpy(), fx[f"bboxes_{b}"], maxulp=2)


@pytest.mark.parametrize("tag", ["retinanet_96x320", "retinanet_288x1280", "retinanet_64x128_nopre"])
def test_against_reference_fixture(tag):
    from visualdet3d_b200 import synth
    fx = load_fixture(tag)
    H, W, B, wseed, iseed, nms_pre = [int(v) for v in fx["meta"]]
    det, _, _ = build(nms_pre=nms_pre)
    img, _ = synth.synth_mono_inputs(B, H, W, seed=iseed)
    res, st = run_with_stages(det, img)
    A, C = det.num_anchors, det.num_classes
    rep = {}
    for i in range(5):
        rep[f"P{i}"] = float(np.abs(subsample_like(st[f"P{i}"], fx[f"P{i}"]) - fx[f"P{i}"]["samples"]).max())
    # head outputs in the reference's concatenated [B, N, C] / [B, N, 4] order (the cls conv's zero padding columns dropped)
    cls = torch.cat([st[f"cls{i}"][:, :A * C].permute(0, 2, 3, 1).reshape(B, -1, C) for i in range(5)], 1)
    reg = torch.cat([st[f"reg{i}"].permute(0, 2, 3, 1).reshape(B, -1, 4) for i in range(5)], 1)
    rep["cls_preds"] = float(np.abs(subsample_like(cls, fx["cls_preds"]) - fx["cls_preds"]["samples"]).max())
    rep["reg_preds"] = float(np.abs(subsample_like(reg, fx["reg_preds"]) - fx["reg_preds"]["samples"]).max())
    print(tag, "stage max|diff| vs reference:", rep, "detections", [len(r[0]) for r in res])
    assert all(v < 1e-3 for v in rep.values()), rep
    for b in range(B):
        s, bx, c = res[b]
        assert len(s) == len(fx[f"scores_{b}"])
        np.testing.assert_array_equal(c.cpu().numpy(), fx[f"cls_{b}"])
        np.testing.assert_allclose(s.cpu().numpy(), fx[f"scores_{b}"], rtol=0, atol=1e-3)
        # box coordinates are pixels: the regression output is scaled by the anchor size (up to ~800 px at P7), so the head-output error
        # (stage tolerance above) enters the boxes multiplied by the box size
        ref = fx[f"bboxes_{b}"]
        size = np.maximum(ref[:, 2] - ref[:, 0], ref[:, 3] - ref[:, 1])[:, None]
        err = np.abs(bx.cpu().numpy() - ref)
        print(tag, "image", b, "max |dbox|", float(err.max()) if err.size else None, "max |dbox| / box size", float((err / size).max()) if err.size else None)
        assert (err <= 1e-3 + 5e-5 * size).all(), err.max()


@pytest.mark.parametrize("B,H,W,cin,cout", [(1, 9, 20, 512, 256), (8, 18, 40, 1024, 256), (2, 3, 5, 2048, 256), (8, 5, 7, 256, 128)])
def test_upsampled_residual_equals_explicit_residual(B, H, W, cin, cout):
    """The fused top-down add (residual read at (y >> 1, x >> 1)) == the same conv with the upsampled tensor as an ordinary residual,
    bit for bit, on ragged sizes (not multiples of the 16 x 8 tile)."""
    from visualdet3d_b200 import engine as E
    g = torch.Generator().manual_seed(B * 100 + H)
    w = torch.randn(cout, cin, 1, 1, generator=g) / cin ** 0.5
    bias = torch.randn(cout, generator=g) * 0.1
    layer = E.ConvLayer(w, bias, None, device="cuda")
    assert layer.engine == "tc16"
    ar = E.Arena()
    x = E.split_lo(E.Act(torch.randn(B, 2 * H, 2 * W, cin, generator=g).cuda(), 0, None,
                         torch.zeros(2, B, 2 * H, 2 * W, cin, dtype=torch.float16, device="cuda")))
    coarse = torch.randn(B, H, W, cout, generator=g).cuda()
    up = coarse.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2).contiguous()
    a = layer(x, ar.act("a", (B, 2 * H, 2 * W, cout), "cuda", lo=True), res=E.Act(coarse), res_up=True)
    b = layer(x, ar.act("b", (B, 2 * H, 2 * W, cout), "cuda", lo=True), res=E.Act(up))
    torch.cuda.synchronize()
    assert torch.equal(a.t, b.t)
    assert torch.equal(a.lo, b.lo)


def test_batch8_equals_single_images_and_graph_replay():
    from visualdet3d_b200 import graphs, synth
    det, _, _ = build()
    img, P2 = synth.synth_mono_inputs(8, 288, 1280, seed=3)
    ic = img.cuda()
    with torch.no_grad():
        r8 = det.forward_batch(ic)
        singles = [det.forward_batch(ic[b:b + 1])[0] for b in range(8)]
        listed = det([ic[:1], None])                    # the reference's list protocol: test_forward, batch 1
    for b in range(8):
        assert all(torch.equal(x, y) for x, y in zip(r8[b], singles[b])), b
    assert all(torch.equal(x, y) for x, y in zip(listed, singles[0])) and listed[2].dtype == torch.int64 and listed[1].shape[1] == 4
    print("detections per image", [len(r[0]) for r in r8])
    # CUDA-graph replay of the step (eager warm-up, capture, replays) == the eager step
    kmax = 256
    rec = torch.zeros(8, 1 + kmax * 13, device="cuda")
    step = graphs.GraphedStep(det, [ic], P2.cuda(), rec, kmax)
    with torch.no_grad():
        step()
        eager = rec.clone()
        step()
        step()
    torch.cuda.synchronize()
    assert step.graph is not None and step.replays >= 1
    assert torch.equal(rec, eager)
    for b in range(8):
        n = int(eager[b, 0])
        assert n == len(r8[b][0])
        rows = eager[b, 1:].view(kmax, 13)[:n]
        assert torch.equal(rows[:, :4], r8[b][1]) and torch.equal(rows[:, 4:11], torch.zeros_like(rows[:, 4:11]))
    with pytest.raises(Exception, match="2-D"):
        graphs.GraphedStep(det, [ic], P2.cuda(), rec, kmax, geometry=True, enabled=False)()


def test_in_place_batchnorm_statistic_refolds_the_plan():
    """Scaling a BatchNorm running_var in place re-folds the weights on the next launch: its outputs equal a freshly built detector loaded
    with the changed state, and differ from the outputs before the change."""
    from visualdet3d_b200 import synth
    det, _, _ = build()
    img, _ = synth.synth_mono_inputs(2, 96, 320, seed=1)
    res0, st0 = run_with_stages(det, img)
    with torch.no_grad():
        det.core.backbone.bn1.running_var.mul_(2.0)
    res1, st1 = run_with_stages(det, img)
    fresh, _, _ = build()
    fresh.load_state_dict(det.state_dict())
    res2, st2 = run_with_stages(fresh, img)
    assert sorted(st1) == sorted(st2)
    assert all(torch.equal(st1[k], st2[k]) for k in st1)
    assert all(torch.equal(x, y) for a, b in zip(res1, res2) for x, y in zip(a, b))
    assert not torch.equal(st1["cls0"], st0["cls0"])


@pytest.mark.parametrize("B", [1, 8])
@pytest.mark.parametrize("cout", [256, 128, 36, 32])
@pytest.mark.parametrize("with_res", [False, True])
def test_multilevel_launch_equals_per_level_launches(B, cout, with_res):
    """One multi-level vd3d_conv2d_tc16 launch over ragged levels (sizes not multiples of the 16 x 8 tile) == the same conv launched level by level,
    bit for bit in the fp32 output and both fp16 planes; with_res: every level adds a half-resolution residual read nearest-upsampled."""
    from visualdet3d_b200 import engine as E
    g = torch.Generator().manual_seed(7 * B + cout + with_res)
    cin = 256
    layer = E.ConvLayer(torch.randn(cout, cin, 3, 3, generator=g) / (9 * cin) ** 0.5, torch.randn(cout, generator=g) * 0.1, None,
                        pad=1, relu=not with_res, device="cuda")
    assert layer.engine == "tc16"
    hws = [(10, 34), (6, 18), (2, 6)] if with_res else [(13, 37), (7, 19), (4, 10), (2, 5), (1, 3)]
    ar = E.Arena()

    def planes_act(h, w, c):
        return E.split_lo(E.Act(torch.randn(B, h, w, c, generator=g).cuda(), 0, None, torch.zeros(2, B, h, w, c, dtype=torch.float16, device="cuda")))
    xs = [planes_act(h, w, cin) for h, w in hws]
    res = None
    if with_res:
        res = ar.level_acts("res", B, [(h // 2, w // 2) for h, w in hws], cout, "cuda")
        for r in res:
            r.t.copy_(torch.randn(r.t.shape, generator=g))
    grouped = layer.run_levels(xs, ar.level_acts("grouped", B, hws, cout, "cuda", lo=True), res=res, res_up=with_res)
    for l, (x, (h, w)) in enumerate(zip(xs, hws)):
        ref = ar.act(f"ref{l}", (B, h, w, cout), "cuda", lo=True)
        layer(x, ref, res=res[l] if with_res else None, res_up=with_res)
        torch.cuda.synchronize()
        assert torch.equal(grouped[l].t, ref.t), l
        assert torch.equal(grouped[l].lo[0], ref.lo[0]) and torch.equal(grouped[l].lo[1], ref.lo[1]), l
