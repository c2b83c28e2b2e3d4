"""-m gpu: the device decode, sort and NMS stages on constructed candidate sets (tests/test_decode_nms_edges_cpu.py builds them and checks
them on the CPU): candidate counts at the kernels' block and capacity edges, score ties, IoU exactly at the threshold, degenerate boxes,
plateau peaks.  These kernels pick index sets, so kept indices, their order and labels must match exactly, and scores and box columns
0..3 bit for bit."""
import numpy as np
import pytest
import torch

from test_decode_nms_edges_cpu import (CHAIN_BOUNDS, CN_H, CN_K, CN_NCLS, CN_W, COUNTS, NCLS_3D, SCORE_THR_3D, anchor_case, chain_image,
                                       cn_cases, cn_maps, cn_oracle, cn_P2, cn_restate, degenerate_image, iou_image, oracle_3d,
                                       plain_image, retina_cases, retina_restate, tie_image)

pytestmark = pytest.mark.gpu


def bits(t):
    return t.contiguous().view(torch.int32)


# ---------------------------------------------------------------------------------------------------------------------------------------
# 3-D anchor head: engine.DecodeNms.run against oracle/torch_port.get_bboxes
# ---------------------------------------------------------------------------------------------------------------------------------------
def run_3d(case, thr, cap, dec=None):
    from visualdet3d_b200 import engine as E
    B = case["cls"].shape[0]
    dec = dec or E.DecodeNms(B, cap, "cuda")
    dec.run(case["cls"].cuda(), case["reg"].cuda(), case["anchors"].cuda(), case["mean_std"].cuda(), case["mask"].cuda(), NCLS_3D,
            SCORE_THR_3D, thr, case["img_w"], case["img_h"])
    torch.cuda.synchronize()
    return dec


def check_3d(dec, case, b, thr):
    (rs, rb, rc, ridx), st = oracle_3d(case, b, thr)
    assert int(dec.ncand[b]) == len(st["cand_scores"]) == case["n"][b]
    k = len(rs)
    assert int(dec.count[b]) == k
    assert torch.equal(dec.anchor[b, :k].cpu().long(), ridx), "kept anchor indices / order"
    assert torch.equal(dec.cls[b, :k].cpu(), rc)
    assert torch.equal(bits(dec.scores[b, :k].cpu()), bits(rs))
    bx = dec.boxes[b, :k].cpu()
    assert torch.equal(bits(bx[:, :4]), bits(rb[:, :4]))
    np.testing.assert_allclose(bx[:, 4:].numpy(), rb[:, 4:].numpy(), rtol=0, atol=1e-6)
    return k


@pytest.mark.parametrize("n", COUNTS)
def test_anchor_candidate_counts(n):
    case = anchor_case([plain_image(n, seed=n)], seed=n)
    check_3d(run_3d(case, 0.4, 2048), case, 0, 0.4)


def test_anchor_overflow_in_one_image_of_a_batch():
    from visualdet3d_b200._lib import Vd3dError
    case = anchor_case([plain_image(100, seed=1), plain_image(2049, seed=2), plain_image(300, seed=3)], seed=4)
    dec = run_3d(case, 0.4, 2048)
    assert int(dec.count[1]) == -1 and int(dec.ncand[1]) == 2049
    with pytest.raises(Vd3dError, match="image 1 "):
        dec.results()
    for b in (0, 2):
        assert check_3d(dec, case, b, 0.4) > 0


@pytest.mark.parametrize("cap", [1000, 40])
def test_anchor_capacity_not_a_power_of_two(cap):
    case = anchor_case([plain_image(cap, seed=cap), plain_image(cap + 1, seed=cap + 1), plain_image(cap * 3 // 5, seed=7)], seed=cap)
    dec = run_3d(case, 0.4, cap)
    assert int(dec.count[1]) == -1 and int(dec.ncand[1]) == cap + 1
    for b in (0, 2):
        check_3d(dec, case, b, 0.4)


def test_anchor_capacity_4096():
    case = anchor_case([plain_image(3000, seed=30)], seed=30)
    check_3d(run_3d(case, 0.4, 4096), case, 0, 0.4)


def test_anchor_chains_across_blocks_and_mask_words():
    """staircases linking sorted positions 63/64, 127/128, 1023/1024 and 2047/2048 (the second suppression word of a lane): in image 0
    the kept box sits before each boundary, in image 1 after it"""
    ims = [chain_image(2100, lambda B: B - 3)[0], chain_image(2100, lambda B: B - 2)[0]]
    case = anchor_case(ims, seed=5)
    dec = run_3d(case, 0.4, 4096)
    for b in range(2):
        assert check_3d(dec, case, b, 0.4) == 2100 - 3 * len(CHAIN_BOUNDS)


def test_anchor_tied_scores_keep_the_lower_index():
    case = anchor_case([tie_image()], seed=2)
    check_3d(run_3d(case, 0.4, 2048), case, 0, 0.4)


@pytest.mark.parametrize("thr", [0.4, 0.5])
def test_anchor_iou_at_the_threshold(thr):
    """IoU = float32(thr) and one ulp either side; 0.4 is not a float32, so float32(0.4) > 0.4 suppresses (torchvision compares the
    float IoU with the double threshold)"""
    im, want = iou_image(thr)
    case = anchor_case([im], seed=9)
    dec = run_3d(case, thr, 2048)
    check_3d(dec, case, 0, thr)
    kept = set(dec.anchor[0, :int(dec.count[0])].cpu().tolist())
    assert [int(case["pos"][0][2 * i + 1]) not in kept for i in range(3)] == want


def test_anchor_degenerate_boxes():
    case = anchor_case([degenerate_image()], img_wh=(200.0, 100.0), seed=4, n_extra=0)
    check_3d(run_3d(case, 0.4, 64), case, 0, 0.4)


def test_anchor_decoder_reuse_with_shrinking_counts():
    dec = None
    for n in (1500, 700, 64, 1, 0):
        case = anchor_case([plain_image(n, seed=100 + n)], seed=100 + n)
        dec = run_3d(case, 0.4, 2048, dec)
        check_3d(dec, case, 0, 0.4)


# ---------------------------------------------------------------------------------------------------------------------------------------
# RetinaNet: RetinaDecode.run_levels against the host restatement (selection by (score desc, anchor index asc))
# ---------------------------------------------------------------------------------------------------------------------------------------
RETINA = retina_cases()


@pytest.mark.parametrize("name", list(RETINA))
def test_retina_decode(name):
    from visualdet3d_b200.detectors.retinanet import RetinaDecode
    c, nms_pre, score_thr, iou_thr = RETINA[name]
    N = c["N"]
    cap = nms_pre if 0 < nms_pre < N else N
    dec = RetinaDecode(c["B"], N, cap, "cuda")
    dec.run_levels([t.cuda() for t in c["cls_lv"]], [t.cuda() for t in c["reg_lv"]], c["level_pix"], c["cls_cs"], c["reg_cs"],
                   c["anchors"].cuda(), c["A"], c["C"], nms_pre, [0.0] * 4, [1.0] * 4, score_thr, iou_thr)
    out = dec.results()
    for b in range(c["B"]):
        rs, rb, rl, ridx = retina_restate(c["cls"][b], c["reg"][b], c["anchors"], nms_pre, [0.0] * 4, [1.0] * 4, score_thr, iou_thr)
        k = len(rs)
        assert int(dec.ncand[b]) == cap
        assert len(out[b][0]) == k > 0
        assert torch.equal(dec.anchor[b, :k].cpu().long(), ridx), "kept anchor indices / order"
        assert torch.equal(out[b][2].cpu(), rl)
        assert torch.equal(bits(out[b][0].cpu()), bits(rs))
        assert torch.equal(bits(out[b][1][:, :4].cpu()), bits(rb))
        assert not bool(out[b][1][:, 4:].any())


# ---------------------------------------------------------------------------------------------------------------------------------------
# CenterNet: MonoFlex / KM3D decode_maps against the documented peak rule, and the oracle's rows
# ---------------------------------------------------------------------------------------------------------------------------------------
_DETS = {}


def centernet(kind):
    if kind not in _DETS:
        from visualdet3d_b200.detectors import build_synthetic_monoflex
        _DETS[kind] = build_synthetic_monoflex(seed=0, name=kind)[0].cuda().eval()
    return _DETS[kind]


def maps_to_act(det, maps):
    from visualdet3d_b200 import engine as E
    pl = det.prepare()
    B = next(iter(maps.values())).shape[0]
    t = torch.zeros(B, CN_H, CN_W, pl["out_channels"])
    for n, v in maps.items():
        t[..., pl["offsets"][n]:pl["offsets"][n] + v.shape[1]] = v.permute(0, 2, 3, 1)
    return E.Act(t.cuda().contiguous())


@pytest.mark.parametrize("kind", ["MonoFlex", "KM3D"])
@pytest.mark.parametrize("name", list(cn_cases()))
def test_centernet_decode(kind, name):
    from visualdet3d_b200._lib import Vd3dError
    peaks, fill, tie_free, _ = cn_cases()[name]
    det = centernet(kind)
    thr, iou = float(det.test_cfg.get("score_thr", 0.1)), float(det.test_cfg.get("nms_iou_thr", 0.5))
    maps = cn_maps(kind, peaks, seed=1, hm_fill=fill)
    B = len(peaks)
    with torch.no_grad():
        dec = det.decode_maps(maps_to_act(det, maps), cn_P2(B).cuda(), 4 * CN_H, 4 * CN_W)
    torch.cuda.synchronize()
    if fill is not None:
        with pytest.raises(Vd3dError, match="image 0 "):
            dec.results()
        assert int(dec.count[0]) == -1 and int(dec.ncand[0]) == CN_NCLS * CN_H * CN_W
    for b in range(B):
        if fill is not None and fill[b] is not None:
            continue
        s, flat, bx = cn_restate(kind, maps, b, thr, iou)
        k = len(s)
        assert int(dec.count[b]) == k > 0
        got = dec.anchor[b, :k].cpu().long()
        assert torch.equal(got, flat), "kept peak indices / order (score desc, flat index asc)"
        assert torch.equal(dec.cls[b, :k].cpu(), flat // (CN_H * CN_W))
        assert torch.equal(bits(dec.scores[b, :k].cpu()), bits(s))
        gb = dec.boxes[b, :k].cpu()
        assert torch.equal(bits(gb[:, :4]), bits(bx))
        rs, rb, rc, rflat = cn_oracle(kind, maps, b, thr, iou)
        if tie_free:
            assert torch.equal(got, rflat)
        rows = {int(f): i for i, f in enumerate(rflat.tolist())}
        common = [(i, rows[int(f)]) for i, f in enumerate(got.tolist()) if int(f) in rows]
        assert len(common) >= k // 2
        gi, ri = torch.tensor([i for i, _ in common]), torch.tensor([j for _, j in common])
        ref = rb[ri]
        np.testing.assert_allclose(gb[gi].numpy(), ref.numpy(), rtol=1e-3, atol=1e-3)
        assert len(s) <= CN_K
