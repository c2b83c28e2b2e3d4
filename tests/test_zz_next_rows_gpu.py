"""-m gpu (runs last): the SURVEY 8(f) "next" rows on the GPU — `test_cfg.post_optimization` on the detector path, the CUDA form of the
hill climbing and of the input pipeline against their host forms (which tests/test_postopt_cpu.py / test_preprocess_cpu.py pin to the reference)."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def wrapped_abs_diff(a, b):
    d = (a - b).abs()
    return torch.minimum(d, (d - 2 * np.pi).abs())


def test_detector_flag_runs_device_post_optimisation():
    """Yolo3D with head.test_cfg.post_optimization=True: the yaw refinement runs as a kernel after the NMS (no host pass) and equals the
    same forward without it followed by the host form `postopt.post_process` (which tests/test_postopt_cpu.py pins to the reference)."""
    from visualdet3d_b200 import synth, postopt, _lib
    from visualdet3d_b200.detectors import build_synthetic_mono3d
    det, sd, cfg, _ = build_synthetic_mono3d("Yolo3D", seed=0)
    det = det.cuda().eval()
    img, P2 = synth.synth_mono_inputs(2, 96, 320, seed=4)
    with torch.no_grad():
        plain = det.forward_batch(img.cuda(), P2.cuda())
        det.post_optimization = True
        try:
            n0 = _lib.launch_count()
            dec = det.launch(img.cuda(), P2.cuda())
            assert _lib.launch_count() > n0
            refined = det.results(dec)
        finally:
            det.post_optimization = False
    changed = 0
    for b, ((s, bx, c), (rs, rb, rc)) in enumerate(zip(plain, refined)):
        assert torch.equal(s, rs) and torch.equal(c, rc) and rb.device == bx.device
        want = postopt.post_process(bx, c, P2[b].numpy()) if len(s) else bx.cpu()
        assert torch.equal(rb.cpu()[:, :10], want[:, :10])
        if len(s):
            assert float(wrapped_abs_diff(rb.cpu()[:, 10], want[:, 10]).max()) < 1e-5
            changed += int((rb.cpu()[:, 10] != bx.cpu()[:, 10]).sum())
    assert changed > 0


def test_device_hill_climbing_matches_reference():
    """vd3d_post_opt (one thread per detection, in place on the fixed-capacity NMS layout) against the UNMODIFIED reference's own outputs
    (tests/golden/postopt.npz: `post_opt` of R/lib/fast_utils/hill_climbing.py run through numba) and against the host form.  Same
    float64 search compiled without FMA contraction; the only differences are last-bit ones of cos / sin / atan2 between the device
    and the host libm, which can move the result by an ulp of float32 but must not change a branch: every row within 1e-5 rad."""
    import os
    from conftest import GOLDEN
    from visualdet3d_b200 import postopt, _lib
    fx = np.load(os.path.join(GOLDEN, "postopt.npz"))
    P2 = fx["P2"]
    P2d = torch.from_numpy(P2).view(1, 3, 4).cuda().contiguous()
    n_cases = len([k for k in fx.files if k.endswith("_in")])
    for ci in range(n_cases):
        b = torch.from_numpy(fx[f"c{ci}_in"])
        labels = torch.from_numpy(fx[f"c{ci}_labels"]).long()
        ref = torch.from_numpy(fx[f"c{ci}_out"])
        host = postopt.post_process(b, labels, P2)
        K = b.shape[0]
        cap = 256
        boxes = torch.zeros(1, cap, 11)
        boxes[0, :K] = b
        cls = torch.zeros(1, cap, dtype=torch.int64)
        cls[0, :K] = labels
        boxes, cls = boxes.cuda(), cls.cuda()
        count = torch.tensor([K], dtype=torch.int32, device="cuda")
        _lib.call("vd3d_post_opt", boxes.data_ptr(), cls.data_ptr(), count.data_ptr(), P2d.data_ptr(), 1, cap, 1280.0, 288.0, 0.4, 0.01, 3.0, 0,
                  torch.cuda.current_stream().cuda_stream)
        got = boxes[0, :K].cpu()
        assert torch.equal(got[:, :10], ref[:, :10])
        assert float(boxes[0, K:].abs().max()) == 0.0                       # rows beyond the count untouched
        sel = (b[:, 6] > 3) & (labels == 0)
        assert torch.equal(got[~sel], b[~sel])                              # unselected rows untouched
        d_ref, d_host = wrapped_abs_diff(got[:, 10], ref[:, 10]), wrapped_abs_diff(got[:, 10], host[:, 10])
        print(f"case {ci}: {int(sel.sum())} refined rows; vs reference: max |d alpha| {float(d_ref.max()):.3g}, bit-identical "
              f"{int((got[sel, 10] == ref[sel, 10]).sum())}; vs host form: max {float(d_host.max()):.3g}")
        assert float(d_host.max()) < 1e-5, d_host
        # the host form itself is bit-identical to the reference on >= 98 % of rows (a last-bit IoU tie can flip a decision in numba's
        # own code path, test_postopt_cpu.py); rows where host == reference must also match the reference on the device
        same = host[:, 10] == ref[:, 10]
        assert float(d_ref[same].max()) < 1e-5


def test_device_post_forward_matches_reference():
    """vd3d_post_forward against the UNMODIFIED reference's BackProjection / BBox3dProjector / 2-D rescale outputs
    (tests/golden/postforward.npz): x, y and the rescaled boxes bit-exact (float32 +,-,*,/ in the reference's order), theta / corners
    through atan2 / cos / sin within float32 rounding."""
    import os
    from conftest import GOLDEN
    from visualdet3d_b200 import engine as E
    fx = np.load(os.path.join(GOLDEN, "postforward.npz"))
    n = len({k.split("_")[0] for k in fx.files})
    seen = 0
    for ci in range(n):
        c = {k[len(f"c{ci}_"):]: fx[k] for k in fx.files if k.startswith(f"c{ci}_")}
        K = len(c["scores"])
        cap = 256
        dec = E.DecodeNms(2, cap, "cuda")                                   # image 0 = the case, image 1 = empty
        dec.boxes.zero_(), dec.scores.zero_(), dec.cls.zero_()
        dec.boxes[0, :K] = torch.from_numpy(c["bbox"]).cuda()
        dec.count.copy_(torch.tensor([K, 0], dtype=torch.int32))
        P2 = torch.from_numpy(np.stack([c["P2"], c["P2"]])).cuda().contiguous()
        oP = torch.from_numpy(np.stack([c["oP"], c["oP"]])).cuda().contiguous()
        dec.post_forward(P2, oP, corners=True)
        assert np.array_equal(dec.box3d[0, :K].cpu().numpy(), c["box3d"]), ci
        assert np.array_equal(dec.box2d[0, :K].cpu().numpy(), c["box2d"]), ci
        if K:
            np.testing.assert_allclose(dec.theta[0, :K].cpu().numpy(), c["thetas"], atol=1e-6, rtol=0)
            np.testing.assert_allclose(dec.corners[0, :K].cpu().numpy(), c["corners"], atol=2e-5, rtol=1e-6)
            np.testing.assert_allclose(dec.homo[0, :K].cpu().numpy(), c["homo"], atol=2e-3, rtol=2e-5)
            seen += K
        assert float(dec.box3d[0, K:].abs().max()) == 0.0 and float(dec.box3d[1].abs().max()) == 0.0
        dec.post_forward(P2, None)                                          # no original_P: boxes copied
        assert torch.equal(dec.box2d[0, :K], dec.boxes[0, :K, :4])
    assert seen > 200


def test_streamed_pipeline_mono_with_post_opt_geometry_and_frames():
    """StreamedInference on a mono detector with `post_optimization` (the GAC config, BASELINE configs[2]): (a) float32 inputs with the
    device geometry columns == `forward_batch` + the host post-forward functions; (b) uint8 frames through the device input pipeline ==
    the same frames preprocessed by `preprocess_batch` and run through `forward_batch`."""
    import os
    import sys
    from conftest import GOLDEN
    sys.path.insert(0, GOLDEN)
    from make_golden_preprocess import frame
    from visualdet3d_b200 import synth, postforward as pf, preprocess as pp
    from visualdet3d_b200.detectors import build_synthetic_mono3d
    from visualdet3d_b200.pipeline import StreamedInference
    det, sd, cfg, _ = build_synthetic_mono3d("Yolo3D", seed=0)
    det = det.cuda().eval()
    det.post_optimization = True
    B, H, W = 2, 96, 320
    img, P2 = synth.synth_mono_inputs(B, H, W, seed=4)
    oP = P2.clone()
    oP[:, :2] *= 1.25
    pipe = StreamedInference(det, B, H, W, kmax=256, geometry=True)
    t = pipe.submit(img.pin_memory(), P2.pin_memory(), original_P=oP.pin_memory())
    pipe.wait_copied(t)
    got = pipe.collect(t)
    with torch.no_grad():
        ref = det.forward_batch(img.cuda(), P2.cuda())
    n = 0
    for b in range(B):
        for x, y in zip(got[b], ref[b]):
            assert torch.equal(x, y.cpu())
        box3d, theta, box2d = pipe.last_geometry[b]
        bx = ref[b][1].cpu()
        want3 = pf.back_projection(bx[:, 4:], P2[b].numpy())
        assert torch.equal(box3d, want3)
        assert torch.equal(box2d, pf.rescale_boxes_2d(bx[:, :4], P2[b].numpy(), oP[b].numpy()))
        if len(bx):
            np.testing.assert_allclose(theta.numpy(), pf.alpha_to_theta(want3[:, 6], want3[:, 0], want3[:, 2], P2[b].numpy()).numpy(), atol=1e-6)
        n += len(bx)
    assert n > 0
    texts = pipe.kitti_text(got, ["Car", "Pedestrian", "Cyclist"], threshold=0.0)
    assert sum(tx.count("\n") for tx in texts) == n
    with pytest.raises(TypeError):
        pipe.submit(img.pin_memory(), img.pin_memory(), P2.pin_memory())     # a mono detector takes one image per sample
    # (b) uint8 frames: 375 x 1242 camera frames -> crop 100 -> 288 x 1280 (the reference's test-time augmentation of the mono configs)
    det.post_optimization = False
    frames = [frame(0, 375, 1242), frame(1, 375, 1242)]
    Hn, Wn = 288, 1280
    pipe2 = StreamedInference(det, 2, Hn, Wn, kmax=256, frame_hw=(375, 1242), crop_top=100)
    _, P2n = synth.synth_mono_inputs(2, Hn, Wn, seed=2)
    fr = torch.from_numpy(np.stack(frames)).pin_memory()
    t = pipe2.submit_frames(fr, P2n.pin_memory())
    got = pipe2.collect(t)
    with torch.no_grad():
        x = pp.preprocess_batch(frames, 100, (Hn, Wn))
        ref = det.forward_batch(x, P2n.cuda())
    for b in range(2):
        for a, r in zip(got[b], ref[b]):
            assert torch.equal(a, r.cpu())
    assert pipe2.h2d_bytes_frames < pipe2.h2d_bytes / 3        # 375 x 1242 x 3 bytes vs 288 x 1280 x 3 floats per frame


def test_graphed_step_replays_the_eager_step_bit_for_bit():
    """graphs.GraphedStep: forward .. NMS + yaw post-optimisation + geometry + record block captured into one CUDA graph; replays over
    refilled static buffers give exactly the record block of the eager launches, and a parameter change drops the stale graph."""
    from visualdet3d_b200 import synth, parallel
    from visualdet3d_b200.detectors import build_synthetic_mono3d
    from visualdet3d_b200.graphs import GraphedStep
    det, sd, cfg, _ = build_synthetic_mono3d("Yolo3D", seed=0)
    det = det.cuda().eval()
    det.post_optimization = True
    B, H, W, kmax = 2, 96, 320, 256
    img = torch.empty(B, 3, H, W, device="cuda")
    P2 = torch.empty(B, 3, 4, device="cuda")
    oP = torch.empty(B, 3, 4, device="cuda")
    rec = torch.empty(B, 1 + kmax * parallel.REC_GEO, device="cuda")
    step = GraphedStep(det, [img], P2, rec, kmax, geometry=True, original_P=oP)
    ndet = 0
    for it in range(5):
        x, p = synth.synth_mono_inputs(B, H, W, seed=30 + it)
        img.copy_(x), P2.copy_(p), oP.copy_(p)
        with torch.no_grad():
            step()
            got = rec.clone()
            dec = det.launch(img, P2)                         # the eager step on the same inputs
            dec.post_forward(P2, oP)
            want = parallel.pack_records_device(dec, kmax, geometry=True).clone()
        torch.cuda.synchronize()
        assert torch.equal(got, want), it
        ndet += int(want[:, 0].sum())
        if it == 2:
            assert step.graph is not None and step.replays >= 1 and step.launches_per_replay > 10
            with torch.no_grad():
                next(det.parameters()).mul_(1.0)              # bumps the parameter version: the plan is rebuilt and the graph dropped
        if it == 3:
            assert step.graph is None
    assert step.graph is not None and ndet > 0


def test_device_input_pipeline_matches_host():
    """preprocess_batch (the augmentation kernel, frames of two different sizes in one batch) vs preprocess_host on the same frames."""
    import os
    import sys
    from conftest import GOLDEN
    sys.path.insert(0, GOLDEN)
    from make_golden_preprocess import frame
    from visualdet3d_b200 import preprocess as pp
    frames = [frame(0, 375, 1242), frame(1, 370, 1224)]
    want = np.stack([pp.preprocess_host(f, 100, (288, 1280)) for f in frames])
    got = pp.preprocess_batch(frames, 100, (288, 1280)).cpu().numpy()
    assert got.shape == (2, 3, 288, 1280) and np.array_equal(got, want)
