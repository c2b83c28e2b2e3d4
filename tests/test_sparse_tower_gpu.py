"""-m gpu: the anchor head's regression tower on the tiles its candidates reach.  The tile-listed conv (vd3d_conv2d_tc16_tiles) against the
dense conv, bit for bit at the stored pixels, with NaN sentinels that must survive everywhere else; poisoned inputs outside the pixels a stored
pixel reads; the device tile lists (vd3d_reg_tower_tiles, with the candidate pixel map of vd3d_reg_candidates) against the numpy restatement
of tests/tower_tiles_cases.py; and the detections of Stereo3D and GroundAwareYolo3D at the bench shapes with the tiled tower on and off."""
import numpy as np
import pytest
import torch

import tower_tiles_cases as tt

pytestmark = pytest.mark.gpu


def _layer(Cin, Cout, relu, seed=0):
    from visualdet3d_b200 import engine as E
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(Cout, Cin, 3, 3, generator=g, dtype=torch.float64) / np.sqrt(9 * Cin)
    return E.ConvLayer(w, torch.randn(Cout, generator=g, dtype=torch.float64), None, pad=1, relu=relu, device="cuda")


def _act(t, planes_only=False):
    """fp32 tensor -> Act with fresh fp16 (hi, lo) planes (planes_only: the fp32 tensor is not valid)"""
    from visualdet3d_b200 import engine as E
    B, H, W, C = t.shape
    x = E.split_lo(E.Act(t.contiguous().cuda(), 0, None, torch.zeros(2, B, H, W, C, dtype=torch.float16, device="cuda")))
    if planes_only:
        x.t.fill_(float("nan"))
        x.f32 = False
    return x


def _nan_out(B, H, W, C):
    from visualdet3d_b200 import engine as E
    return E.Act(torch.full((B, H, W, C), float("nan"), device="cuda"), 0, None,
                 torch.full((2, B, H, W, C), float("nan"), dtype=torch.float16, device="cuda"))


def _device_list(cand, d):
    """numpy tile list of depth d -> (list [cap, 4], count [1], store map [B, H, W]) on the device; entries past the count are garbage"""
    B, H, W = cand.shape
    s, lst = tt.tiles(cand, d)
    t = torch.full((tt.cap(B, H, W), 4), -12345, dtype=torch.int32)
    t[:len(lst)] = torch.from_numpy(lst)
    return t.cuda(), torch.tensor([len(lst)], dtype=torch.int32).cuda(), torch.from_numpy(s.astype(np.uint8)).cuda()


def _run(layer, x, res, f32_out, cand, d):
    """(dense output, tile-listed output, store map [B, H, W] bool on the CPU)"""
    from visualdet3d_b200 import engine as E
    B, H, W = x.B, x.H, x.W
    dense = layer(x, _nan_out(B, H, W, layer.Cout), res=res, f32_out=f32_out)
    tiles = _device_list(cand, d)
    out = layer(x, _nan_out(B, H, W, layer.Cout), res=res, f32_out=f32_out, tiles=tiles)
    torch.cuda.synchronize()
    assert out.valid is tiles[2]
    return dense, out, tiles[2].bool().cpu()


def _assert_stored(dense, out, smap, f32_out):
    """bit-identical at the store map, the NaN sentinels untouched elsewhere (both planes, and the fp32 tensor when written)"""
    forms = [(dense.lo[0], out.lo[0]), (dense.lo[1], out.lo[1])] + ([(dense.t, out.t)] if f32_out else [])
    for dn, ot in forms:
        dn, ot = dn.cpu(), ot.cpu()
        assert torch.equal(ot[smap].view(torch.int16 if ot.dtype == torch.float16 else torch.int32),
                           dn[smap].view(torch.int16 if dn.dtype == torch.float16 else torch.int32)), "stored pixels differ from the dense conv"
        assert torch.isnan(ot[~smap]).all(), "the tile-listed conv stored outside its map"
    if not f32_out:
        assert torch.isnan(out.t.cpu()).all(), "a planes-only launch wrote the fp32 tensor"


MAPS = tt.maps()
# (map, depth): empty, one pixel at each image corner, bands at the top and bottom edges, every tile, candidates in every image, W % 16 != 0
LISTS = [("empty", 1), ("corners", 1), ("corners", 3), ("edge_bands", 2), ("full", 1), ("bench_like", 3), ("dense_random", 1), ("ragged", 2)]


@pytest.mark.parametrize("name,d", LISTS, ids=[f"{n}-d{d}" for n, d in LISTS])
@pytest.mark.parametrize("Cout", [256, 140, 64], ids=["n128", "ntail", "n64"])
def test_tile_listed_conv_matches_dense(name, d, Cout):
    """fp32 + planes output, ReLU, no residual; Cout 256 (128-column tiles on the epilogue warps), 140 (a Cout % 8 == 4 tail column group),
    64 (the consumer-run epilogue)"""
    cand = MAPS[name]
    B, H, W = cand.shape
    g = torch.Generator().manual_seed(2)
    x = _act(torch.randn(B, H, W, 128, generator=g))
    layer = _layer(128, Cout, relu=True)
    dense, out, smap = _run(layer, x, None, True, cand, d)
    _assert_stored(dense, out, smap, True)


@pytest.mark.parametrize("res", ["none", "f32", "planes"])
@pytest.mark.parametrize("f32_out", [True, False], ids=["f32+planes", "planes"])
@pytest.mark.parametrize("relu", [True, False], ids=["relu", "linear"])
def test_tile_listed_conv_residual_and_output_forms(res, f32_out, relu):
    cand = MAPS["bench_like"]
    B, H, W = cand.shape
    g = torch.Generator().manual_seed(4)
    x = _act(torch.randn(B, H, W, 128, generator=g))
    layer = _layer(128, 128, relu=relu, seed=1)
    r = None if res == "none" else _act(torch.randn(B, H, W, 128, generator=g), planes_only=res == "planes")
    dense, out, smap = _run(layer, x, r, f32_out, cand, 2)
    _assert_stored(dense, out, smap, f32_out)


@pytest.mark.parametrize("poison", [float("nan"), 1e30])
def test_poison_outside_the_read_set(poison):
    """Input poisoned outside S_{d+1} and residual outside S_d (what a stored pixel of depth d reads): no stored bit changes and the
    fp16-range guard stays clear"""
    from visualdet3d_b200 import engine as E
    cand = MAPS["bench_like"]
    B, H, W = cand.shape
    d = 2
    g = torch.Generator().manual_seed(6)
    xt, rt = torch.randn(B, H, W, 128, generator=g), torch.randn(B, H, W, 128, generator=g)
    layer = _layer(128, 128, relu=True, seed=3)
    dense = layer(_act(xt), _nan_out(B, H, W, 128), res=_act(rt))
    read = torch.from_numpy(tt.dilate(cand, d + 1))
    xt[~read] = poison
    rt[~torch.from_numpy(tt.dilate(cand, d))] = poison
    x, r = _act(xt), _act(rt)                       # (splitting the poisoned values trips the guard: clear it afterwards)
    torch.cuda.synchronize()
    E.fp16_range_overflowed(reset=True)
    tiles = _device_list(cand, d)
    out = layer(x, _nan_out(B, H, W, 128), res=r, tiles=tiles)
    torch.cuda.synchronize()
    _assert_stored(dense, out, tiles[2].bool().cpu(), True)
    assert not E.fp16_range_overflowed(reset=True), "a pixel outside the store map reached the fp16-range guard"


@pytest.mark.parametrize("name", sorted(MAPS))
def test_device_tile_lists_match_numpy(name):
    """vd3d_reg_candidates' pixel map of constructed scores, then vd3d_reg_tower_tiles for depths 1..3, against tests/tower_tiles_cases.py"""
    from visualdet3d_b200 import engine as E
    cand = MAPS[name]
    B, H, W = cand.shape
    A, ncls = 16, 2
    # one anchor of a candidate pixel scores above the threshold (sigmoid(4) = 0.98), every other anchor far below; anchor 9 (group 1) for
    # odd pixels, anchor 0 (group 0) for even ones, so the pixel map is the union over the groups
    cls = torch.full((B, H * W, A, ncls + 1), -4.0)
    flat = torch.from_numpy(cand.reshape(B, H * W).astype(bool))
    a_of = torch.where(torch.arange(H * W) % 2 == 1, 9, 0)
    for b in range(B):
        idx = torch.nonzero(flat[b]).flatten()
        cls[b, idx, a_of[idx], 1] = 4.0
    mask = torch.ones(B, H * W * A, dtype=torch.uint8, device="cuda")
    groups = A // E.REG_GROUP_ANCHORS
    lst = torch.empty(groups, B * H * W, dtype=torch.int32, device="cuda")
    counts = torch.empty(groups, dtype=torch.int32, device="cuda")
    pix = torch.full((B, H, W), 77, dtype=torch.uint8, device="cuda")
    E.reg_candidates(cls.view(B, H, W, -1).cuda(), mask, A, ncls, 0.5, lst, counts, pix)
    D = 3
    smaps = torch.full((D, B, H, W), 5, dtype=torch.uint8, device="cuda")
    tiles = torch.full((D, E.tower_tile_cap(B, H, W), 4), -1, dtype=torch.int32, device="cuda")
    tcount = torch.full((D,), -1, dtype=torch.int32, device="cuda")
    E.tower_tiles(pix, smaps, tiles, tcount)
    torch.cuda.synchronize()
    assert torch.equal(pix.cpu(), torch.from_numpy(cand.astype(np.uint8)))
    for d in range(1, D + 1):
        s, want = tt.tiles(cand, d)
        n = int(tcount[d - 1])
        assert n == len(want), f"depth {d}"
        assert torch.equal(tiles[d - 1, :n].cpu(), torch.from_numpy(want)), f"depth {d}"
        assert torch.equal(smaps[d - 1].cpu(), torch.from_numpy(s.astype(np.uint8))), f"depth {d}"


def _dets(det, inputs):
    dec = det.launch(*inputs)
    torch.cuda.synchronize()
    return [t.clone() for t in (dec.count, dec.scores, dec.boxes, dec.cls, dec.anchor, dec.ncand)]


@pytest.mark.parametrize("config", ["stereo", "gac"])
def test_detections_identical_tiled_tower_and_dense(config, monkeypatch):
    """the bench shapes at batch 8: the tiled tower is the path taken, and it detects exactly what the fully dense head does"""
    from visualdet3d_b200 import synth
    from visualdet3d_b200.detectors import build_synthetic_mono3d, build_synthetic_stereo3d
    if config == "stereo":
        det = build_synthetic_stereo3d(seed=0)[0]
        l, r, p2, _ = synth.synth_stereo_inputs(8, 384, 1280, seed=1)
        inputs = [l.cuda(), r.cuda(), p2.cuda()]
    else:
        det = build_synthetic_mono3d("GroundAwareYolo3D", seed=0)[0]
        im, p2 = synth.synth_mono_inputs(8, 288, 1280, seed=1)
        inputs = [im.cuda(), p2.cuda()]
    det = det.cuda().eval()
    B, _, H, W = inputs[0].shape
    with torch.no_grad():
        pl = det.prepare()
        assert det.sparse_reg(pl["reg_out"], B, H // 16, W // 16)
        assert det.tower_tiles_ok(det.reg_tower(pl), pl["reg_out"], H // 16, W // 16)
        tiled = _dets(det, inputs)
        n = det._arena.get("tower_count", (len(det.reg_tower(pl)),), inputs[0].device, dtype=torch.int32).cpu()
        dense_tiles = B * -(-(H // 16) // 8) * -(-(W // 16) // 16)
        assert (n > 0).all() and (n <= dense_tiles).all() and bool((n[:-1] <= n[1:]).all())     # deeper convs, larger sets
        monkeypatch.setenv("VD3D_SPARSE_REG", "0")
        dense = _dets(det, inputs)
    count = dense[0].cpu()
    assert int(count.min()) >= 0 and int(count.sum()) > 0
    assert torch.equal(tiled[0], dense[0]) and torch.equal(tiled[5], dense[5])
    for b, k in enumerate(count.tolist()):
        for s, d in zip(tiled[1:5], dense[1:5]):
            assert torch.equal(s[b, :k], d[b, :k]), f"image {b}"
