"""End-to-end parity of the B200 Stereo3D forward (-m gpu) against (a) the committed reference fixtures and
(b) the CPU oracle run on the same seeded inputs.  Tolerances (BASELINE.json north_star): bit-exact anchor
indices / masks / keep sets, scores and boxes within 1e-3 (fp32)."""
import numpy as np
import pytest
import torch

from conftest import load_fixture, subsample_like
import torch_port as tp
from detector_harness import assert_dets_match, run_with_stages

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def det_bundle():
    from visualdet3d_b200.detectors import build_synthetic_stereo3d
    det, sd, cfg, priors = build_synthetic_stereo3d(seed=0)
    return det.cuda().eval(), sd, cfg, priors


@pytest.mark.parametrize("tag", ["stereo3d_96x320", "stereo3d_192x640", "stereo3d_384x1280"])    # the last one = BASELINE configs[1] shape
def test_against_reference_fixture(det_bundle, tag):
    from visualdet3d_b200 import synth
    det, sd, cfg, (pm, ps) = det_bundle
    fx = load_fixture(tag)
    H, W, B, seed = [int(v) for v in fx["meta"]]
    left, right, P2, P3 = synth.synth_stereo_inputs(B, H, W, seed=1)
    res, st = run_with_stages(det, left, right, P2, flatten_heads=True)
    report = {}
    for nm in ["feat4", "vol4", "vol8", "vol16", "features", "cls_preds", "reg_preds"]:
        got = subsample_like(st[nm], fx[nm])
        report[nm] = float(np.abs(got - fx[nm]["samples"]).max())
    print(tag, "stage max|diff| vs reference:", report)
    for nm, v in report.items():
        assert v < 5e-4, (nm, v)
    for b in range(B):
        np.testing.assert_array_equal(np.packbits(st["mask"][b].numpy().astype(bool)), fx[f"mask_{b}"])
        s, bx, ci = [t.cpu() for t in res[b]]
        assert len(s) == len(fx[f"scores_{b}"]), (len(s), len(fx[f"scores_{b}"]))
        np.testing.assert_array_equal(ci.numpy(), fx[f"cls_{b}"])
        np.testing.assert_allclose(s.numpy(), fx[f"scores_{b}"], atol=1e-3, rtol=0)
        np.testing.assert_allclose(bx.numpy(), fx[f"bboxes_{b}"], atol=1e-3, rtol=0)
        assert ci.dtype == torch.int64 and bx.shape[1] == 11


def test_against_oracle_ragged_batch(det_bundle):
    """B = 3 at 128x384 (not a fixture size): stages, masks, keep sets (anchor indices) and outputs vs the oracle."""
    from visualdet3d_b200 import synth
    det, sd, cfg, (pm, ps) = det_bundle
    B, H, W = 3, 128, 384
    left, right, P2, P3 = synth.synth_stereo_inputs(B, H, W, seed=7)
    res, st = run_with_stages(det, left, right, P2, flatten_heads=True)
    ost = {}
    ref = tp.stereo3d_forward(sd, left, right, P2, cfg, pm, ps, ost)
    for nm in ["feat4", "feat8", "feat16", "vol4", "vol8", "vol16", "features", "cls_preds", "reg_preds"]:
        d = float((st[nm] - ost[nm]).abs().max())
        print(nm, "max|diff|", d, "scale", float(ost[nm].abs().mean()))
        assert d < 5e-4, (nm, d)
    assert torch.equal(st["mask"].bool(), ost["mask"])
    dec = det._last_decoder
    for b in range(B):
        s, bx, ci = [t.cpu() for t in res[b]]
        rs, rb, rc, ridx = ref[b]
        assert len(s) == len(rs)
        k = len(s)
        assert torch.equal(dec.anchor[b, :k].cpu().long(), ridx)          # bit-exact kept anchor indices, in NMS order
        assert torch.equal(ci, rc)
        assert float((s - rs).abs().max()) < 1e-3 and float((bx - rb).abs().max()) < 1e-3
        assert bool((s[:-1] >= s[1:]).all())                               # descending scores


def test_decode_nms_exact_on_oracle_predictions(det_bundle):
    """Decode + NMS in isolation, fed with the ORACLE's cls/reg predictions: candidate sets, keep indices and order must
    be bit-exact, values within 1e-4 (libm expf/atan2f ulps)."""
    from visualdet3d_b200 import synth, engine as E
    from visualdet3d_b200.anchors import AnchorTable
    det, sd, cfg, (pm, ps) = det_bundle
    B, H, W = 2, 192, 640
    left, right, P2, P3 = synth.synth_stereo_inputs(B, H, W, seed=3)
    ost = {}
    ref = tp.stereo3d_forward(sd, left, right, P2, cfg, pm, ps, ost)
    tab = AnchorTable((H, W), det.anchors_cfg, pm, ps, "cuda")
    mask = torch.empty(B, tab.N, dtype=torch.uint8, device="cuda")
    E.anchor_mask(tab.anchors, tab.means_z, P2.cuda(), mask)
    assert torch.equal(mask.cpu().bool(), ost["mask"])
    dec = E.DecodeNms(B, 2048, "cuda")
    dec.run(ost["cls_preds"].cuda().contiguous(), ost["reg_preds"].cuda().contiguous(), tab.anchors, tab.mean_std, mask,
            2, 0.75, 0.4, W, H)
    out = dec.results()
    for b in range(B):
        rs, rb, rc, ridx = ref[b]
        k = len(rs)
        assert int(dec.ncand[b]) == len(ost["per_image"][b]["cand_scores"])
        assert len(out[b][0]) == k and k > 5
        assert torch.equal(dec.anchor[b, :k].cpu().long(), ridx)
        assert torch.equal(out[b][2].cpu(), rc)
        np.testing.assert_allclose(out[b][0].cpu().numpy(), rs.numpy(), atol=1e-6)
        np.testing.assert_allclose(out[b][1].cpu().numpy(), rb.numpy(), atol=1e-4)


def test_full_size_batch8_all_images_vs_oracle(det_bundle):
    """BASELINE config[1] shape (batch 8, 384x1280): determinism, batch invariance (image b of the batched run == the same pair
    run alone), and EVERY image of the batch against the oracle (kept anchor sets, order, values within 1e-3)."""
    from visualdet3d_b200 import synth
    det, sd, cfg, (pm, ps) = det_bundle
    B, H, W = 8, 384, 1280
    left, right, P2, P3 = synth.synth_stereo_inputs(B, H, W, seed=11)
    l, r, p = left.cuda(), right.cuda(), P2.cuda()
    with torch.no_grad():
        res = det.forward_batch(l, r, p)
        anchors = [det._last_decoder.anchor[b, :len(res[b][0])].clone() for b in range(B)]
        res2 = det.forward_batch(l, r, p)
        single = det([l[5:6], r[5:6], p[5:6], None])
    for a, b in zip(res, res2):
        assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert all(torch.equal(x, y) for x, y in zip(res[5], single))
    assert sum(len(x[0]) for x in res) > 8
    ref = tp.stereo3d_forward(sd, left, right, P2, cfg, pm, ps)
    swaps = [assert_dets_match(res[b], ref[b], anchors[b]) for b in range(B)]
    print("full-size batch: detections per image", [len(x[0]) for x in res], "score-tied order swaps", swaps)


def test_reference_list_protocol_and_empty_result(det_bundle):
    from visualdet3d_b200 import synth
    det, *_ = det_bundle
    left, right, P2, P3 = synth.synth_stereo_inputs(1, 96, 320, seed=1)
    old = det.test_cfg["score_thr"]
    det.test_cfg["score_thr"] = 0.999999
    try:
        s, b, c = det([left.cuda(), right.cuda(), P2.cuda(), P3.cuda()])
    finally:
        det.test_cfg["score_thr"] = old
    assert s.shape == (0,) and b.shape == (0, 11) and c.shape == (0,) and c.dtype == torch.int64
    with pytest.raises(AssertionError):
        l2, r2, p2, _ = synth.synth_stereo_inputs(2, 96, 320)
        det([l2.cuda(), r2.cuda(), p2.cuda(), None])


def test_lo_companions_are_fresh_everywhere(det_bundle, monkeypatch):
    """VD3D_CHECK_LO: before every tensor-core conv the `lo` tensor must equal t - (t & 0xFFFFE000) (no stale split)."""
    from visualdet3d_b200 import synth, engine
    det, *_ = det_bundle
    monkeypatch.setattr(engine, "CHECK_LO", True)
    left, right, P2, P3 = synth.synth_stereo_inputs(2, 96, 320, seed=4)
    with torch.no_grad():
        det.forward_batch(left.cuda(), right.cuda(), P2.cuda())


def test_engines_agree(det_bundle):
    """The wgmma engines (fp16-split default, 3xTF32) and the exact-fp32 SIMT engine give the same detections (sets) and
    values within 1e-3."""
    import os
    from visualdet3d_b200 import synth
    from visualdet3d_b200.detectors import build_synthetic_stereo3d
    det, sd, cfg, _ = det_bundle
    left, right, P2, P3 = synth.synth_stereo_inputs(2, 192, 640, seed=5)
    with torch.no_grad():
        a = det.forward_batch(left.cuda(), right.cuda(), P2.cuda())
        anchors_a = [det._last_decoder.anchor[b, :len(a[b][0])].cpu() for b in range(2)]
    for eng in ("simt", "tc"):
        os.environ["VD3D_CONV_ENGINE"] = eng
        try:
            det2, *_ = build_synthetic_stereo3d(seed=0)
            det2 = det2.cuda().eval()
            det2.prepare()
        finally:
            os.environ.pop("VD3D_CONV_ENGINE", None)
        with torch.no_grad():
            bres = det2.forward_batch(left.cuda(), right.cuda(), P2.cuda())
            anchors_b = [det2._last_decoder.anchor[b, :len(bres[b][0])].cpu() for b in range(2)]
        for b in range(2):
            assert len(a[b][0]) > 3
            sa, ia = torch.sort(anchors_a[b])
            sb, ib = torch.sort(anchors_b[b])
            assert torch.equal(sa, sb), eng                                    # same kept anchors ...
            for j in (0, 1, 2):                                                # ... and, row for row after aligning on the anchor index,
                va, vb = a[b][j][ia.cuda()], bres[b][j][ib.cuda()]            # the same scores / boxes / classes
                if j == 2:
                    assert torch.equal(va, vb), eng
                else:
                    assert float((va - vb).abs().max()) < 1e-3, (eng, j, float((va - vb).abs().max()))
            moved = (anchors_a[b] != anchors_b[b]).nonzero()[:, 0].tolist()    # order may differ only between score-tied rows
            for i in moved:
                assert abs(float(a[b][0][i]) - float(bres[b][0][i])) < 1e-5, eng


def test_device_record_block_matches_results(det_bundle):
    """parallel.pack_records_device (one kernel, no host sync) == the per-image results, through unpack_records."""
    from visualdet3d_b200 import synth, parallel
    det, *_ = det_bundle
    left, right, P2, P3 = synth.synth_stereo_inputs(3, 128, 384, seed=2)
    with torch.no_grad():
        dec = det.launch(left.cuda(), right.cuda(), P2.cuda())
        rec = parallel.all_gather_records(parallel.pack_records_device(dec, 64))
    ref = dec.results()
    got = parallel.unpack_records(rec.cpu())
    assert len(got) == 3
    for (s, b, c), (rs, rb, rc) in zip(got, ref):
        assert torch.equal(s, rs.cpu()) and torch.equal(b, rb.cpu()) and torch.equal(c, rc.cpu())
    # overflow is flagged, not truncated
    small = parallel.pack_records_device(dec, 1)
    if max(len(r[0]) for r in ref) > 1:
        with pytest.raises(RuntimeError):
            parallel.unpack_records(small.cpu())


def test_streamed_pipeline_matches_forward_batch(det_bundle):
    """visualdet3d_b200.pipeline.StreamedInference (pinned host batches, copy stream, async D2H of the record block): three
    different batches in flight give exactly the detections of `forward_batch` on the same inputs, in submission order."""
    from visualdet3d_b200 import synth
    from visualdet3d_b200.pipeline import StreamedInference
    det = det_bundle[0]
    B, H, W = 2, 96, 320
    pipe = StreamedInference(det, B, H, W, kmax=512)
    batches = [synth.synth_stereo_inputs(B, H, W, seed=20 + i) for i in range(3)]
    pinned = [(l.pin_memory(), r.pin_memory(), p.pin_memory()) for (l, r, p, _) in batches]
    tickets = [pipe.submit(*pinned[0]), pipe.submit(*pinned[1])]
    got = [pipe.collect(tickets[0])]
    tickets.append(pipe.submit(*pinned[2]))
    got += [pipe.collect(tickets[1]), pipe.collect(tickets[2])]
    for (l, r, p, _), g in zip(batches, got):
        with torch.no_grad():
            ref = det.forward_batch(l.cuda(), r.cuda(), p.cuda())
        assert len(g) == B
        for (s, bx, c), (rs, rb, rc) in zip(g, ref):
            assert torch.equal(s, rs.cpu()) and torch.equal(bx, rb.cpu()) and torch.equal(c, rc.cpu())
    with pytest.raises(ValueError):
        pipe.submit(batches[0][0], batches[0][1], batches[0][2])          # not pinned
