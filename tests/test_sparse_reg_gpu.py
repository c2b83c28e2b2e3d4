"""-m gpu: the anchor head's regression conv on the decoder's rows only.  The gathered-row conv (vd3d_conv2d_tc16_gather) against the dense
conv, bit for bit at the listed pixels, on constructed lists; the candidate list (vd3d_reg_candidates) against its definition; and the
detections of Stereo3D, Yolo3D and GroundAwareYolo3D at the bench image sizes, batch 8, with the sparse path on and off."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GROUP = 96          # output columns per list group (8 anchors x 12)


def _layer(Cin, Cout, seed=0):
    from visualdet3d_b200 import engine as E
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(Cout, Cin, 3, 3, generator=g, dtype=torch.float64) / np.sqrt(9 * Cin)
    return E.ConvLayer(w, torch.randn(Cout, generator=g, dtype=torch.float64), None, pad=1, relu=False, device="cuda")


def _input(B, H, W, Cin, seed=1):
    from visualdet3d_b200 import engine as E
    g = torch.Generator().manual_seed(seed)
    x = E.Act(torch.randn(B, H, W, Cin, generator=g).cuda(), 0, None, torch.zeros(2, B, H, W, Cin, dtype=torch.float16, device="cuda"))
    return E.split_lo(x)


def _lists(pairs, groups, npix):
    """[(group, pixel)] -> (list [groups][npix] int32, counts [groups] int32) on the device, each group's pixels in a shuffled order"""
    lst = torch.full((groups, npix), -7, dtype=torch.int32)
    counts = torch.zeros(groups, dtype=torch.int32)
    by = {}
    for grp, p in pairs:
        by.setdefault(grp, []).append(p)
    rng = np.random.default_rng(3)
    for grp, ps in by.items():
        ps = list(rng.permutation(ps))
        lst[grp, :len(ps)] = torch.tensor(ps, dtype=torch.int32)
        counts[grp] = len(ps)
    return lst.cuda(), counts.cuda()


def _check(B, H, W, Cin, Cout, pairs):
    from visualdet3d_b200 import engine as E
    layer = _layer(Cin, Cout)
    x = _input(B, H, W, Cin)
    dense = layer(x, E.Act(torch.empty(B, H, W, Cout, device="cuda")))
    groups = -(-Cout // GROUP)
    lst, counts = _lists(pairs, groups, B * H * W)
    out = E.Act(torch.full((B, H, W, Cout), float("nan"), device="cuda"))
    layer.gather(x, lst, counts, out)
    torch.cuda.synchronize()
    want = torch.zeros(B * H * W, Cout, dtype=torch.bool)
    for grp, p in pairs:
        want[p, grp * GROUP:(grp + 1) * GROUP] = True
    got = out.t.view(-1, Cout).cpu()
    ref = dense.t.view(-1, Cout).cpu()
    assert torch.equal(got[want], ref[want]), "gathered rows differ from the dense conv"
    assert torch.isnan(got[~want]).all(), "the gathered conv wrote outside its list"


SHAPE = (2, 6, 20)          # B, H, W: 240 pixels, two images


def _all_pixels(groups, npix):
    return [(g, p) for g in range(groups) for p in range(npix)]


def _border(B, H, W, groups):
    return [(g, (b * H + h) * W + w) for g in range(groups) for b in range(B) for h in range(H) for w in range(W)
            if h in (0, H - 1) or w in (0, W - 1)]


@pytest.mark.parametrize("Cin,Cout", [(128, 576), (136, 432), (1408, 576)])
@pytest.mark.parametrize("case", ["empty", "one", "border", "ragged", "across_images", "all"])
def test_gathered_conv_matches_dense(case, Cin, Cout):
    B, H, W = SHAPE
    groups, npix = -(-Cout // GROUP), B * H * W
    if case == "empty":
        pairs = []
    elif case == "one":
        pairs = [(groups - 1, npix // 2 + 3)]
    elif case == "border":
        pairs = _border(B, H, W, groups)
    elif case == "ragged":                   # two tiles in group 1 (the second with 2 rows), one partial tile in group 0
        pairs = [(1, p) for p in range(130)] + [(0, p) for p in range(5, npix, 7)]
    elif case == "across_images":
        pairs = [(g, b * H * W + (5 * g + 11 * b) % (H * W)) for g in range(groups) for b in range(B)] + [(0, H * W - 1), (0, H * W)]
    else:                                    # every anchor a candidate: the list at its capacity
        pairs = _all_pixels(groups, npix)
    _check(B, H, W, Cin, Cout, pairs)


def test_reg_candidates_definition():
    """pair (b, pixel, group) listed iff some anchor of the group is in the mask and its best class clears the threshold"""
    from visualdet3d_b200 import engine as E
    B, P, A, ncls, thr = 3, 77, 48, 2, 0.75
    g = torch.Generator().manual_seed(5)
    # logits far from the threshold (sigmoid(+-4) = 0.982 / 0.018): the test does not depend on the last bit of the sigmoid
    cls = torch.where(torch.rand(B, P, 1, A * (ncls + 1), generator=g) < 0.02, 4.0, -4.0).cuda()
    mask = (torch.rand(B, P * A, generator=g) < 0.4).to(torch.uint8).cuda()
    groups = A // E.REG_GROUP_ANCHORS
    lst = torch.full((groups, B * P), -1, dtype=torch.int32, device="cuda")
    counts = torch.full((groups,), 999, dtype=torch.int32, device="cuda")
    E.reg_candidates(cls, mask, A, ncls, thr, lst, counts)
    torch.cuda.synchronize()
    c = cls.view(B, P, A, ncls + 1)[..., :ncls].cpu()
    hit = (torch.sigmoid(c).max(-1).values > thr) & mask.view(B, P, A).bool().cpu()
    want = hit.view(B * P, groups, E.REG_GROUP_ANCHORS).any(-1)            # [B * P, groups]
    counts, lst = counts.cpu(), lst.cpu()
    for grp in range(groups):
        n = int(counts[grp])
        got = sorted(lst[grp, :n].tolist())
        assert got == torch.nonzero(want[:, grp]).flatten().tolist(), f"group {grp}"
    assert int(counts.sum()) > 0


def _dets(det, inputs):
    dec = det.launch(*inputs)
    torch.cuda.synchronize()
    return [t.clone() for t in (dec.count, dec.scores, dec.boxes, dec.cls, dec.anchor, dec.ncand)]


@pytest.mark.parametrize("config", ["stereo", "gac", "yolo3d"])
def test_detections_identical_sparse_and_dense(config, monkeypatch):
    """(batch 8 for all three: Yolo3D's bench batch of 1 keeps the dense conv, see Anchor3DDetector.sparse_reg)"""
    from visualdet3d_b200 import synth
    from visualdet3d_b200.detectors import build_synthetic_mono3d, build_synthetic_stereo3d
    if config == "stereo":
        det = build_synthetic_stereo3d(seed=0)[0]
        l, r, p2, _ = synth.synth_stereo_inputs(8, 384, 1280, seed=1)
        inputs = [l.cuda(), r.cuda(), p2.cuda()]
    else:
        det = (build_synthetic_mono3d("GroundAwareYolo3D", seed=0) if config == "gac" else build_synthetic_mono3d("Yolo3D", seed=0, depth=18))[0]
        im, p2 = synth.synth_mono_inputs(8, 288, 1280, seed=1)
        inputs = [im.cuda(), p2.cuda()]
    det = det.cuda().eval()
    B, _, H, W = inputs[0].shape
    with torch.no_grad():
        assert det.sparse_reg(det.prepare()["reg_out"], B, H // 16, W // 16)
        sparse = _dets(det, inputs)
        monkeypatch.setenv("VD3D_SPARSE_REG", "0")
        dense = _dets(det, inputs)
    count = dense[0].cpu()
    assert int(count.min()) >= 0 and int(count.sum()) > 0
    assert torch.equal(sparse[0], dense[0]) and torch.equal(sparse[5], dense[5])
    for b, k in enumerate(count.tolist()):
        for s, d in zip(sparse[1:5], dense[1:5]):
            assert torch.equal(s[b, :k], d[b, :k]), f"image {b}"
