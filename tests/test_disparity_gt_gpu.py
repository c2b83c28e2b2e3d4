"""GPU checks of Stereo3D's disparity ground truth (csrc/disparity_gt.cu) against tests/golden/disparity_gt.npz (cv2 and the unmodified
reference): StereoBM and the reduced maps bit for bit on every case and in batches, the float32 front end, the LiDAR maps, CUDA graph
replay, input checks, and the precompute CLI over a constructed KITTI tree in both modes."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from conftest import ROOT, load_fixture
import disparity_gt_cases as dc
import stereo_bm as sb

pytestmark = pytest.mark.gpu
CASES = {c["id"]: c for c in dc.bm_cases()}


@pytest.fixture(scope="module")
def fx():
    return load_fixture("disparity_gt")


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("cid", list(CASES))
def test_stereo_bm_equals_golden(cid, fx):
    from visualdet3d_b200 import disparity_gt as dg
    c = CASES[cid]
    d = dg.stereo_bm(_dev(c["left"][None]), _dev(c["right"][None]))
    torch.cuda.synchronize()
    np.testing.assert_array_equal(d[0].cpu().numpy(), fx["bm"][cid])
    np.testing.assert_array_equal(dg.block_max(d)[0].cpu().numpy(), fx["bmr"][cid])


def _crop_batch(shape):
    H, W = shape
    ids = [k for k, c in CASES.items() if c["left"].shape[0] >= H and c["left"].shape[1] >= W]
    return ids, np.stack([CASES[k]["left"][:H, :W] for k in ids]), np.stack([CASES[k]["right"][:H, :W] for k in ids])


@pytest.mark.parametrize("shape", [(64, 400), (26, 216), (97, 451)])
def test_mixed_batch_equals_cv2(shape):
    cv2 = pytest.importorskip("cv2")
    from visualdet3d_b200 import disparity_gt as dg
    ids, L, R = _crop_batch(shape)
    assert len(ids) >= 3
    d = dg.stereo_bm(_dev(L), _dev(R)).cpu().numpy()
    m = cv2.StereoBM_create(192, 25)
    for b in range(len(ids)):
        ref = m.compute(L[b], R[b])
        np.testing.assert_array_equal(d[b], ref, err_msg=ids[b])


def test_large_shapes_batched(fx):
    from visualdet3d_b200 import disparity_gt as dg
    c = CASES["shape_288x1280"]
    L = np.stack([c["left"], c["right"], c["left"]])
    R = np.stack([c["right"], c["left"], c["right"]])
    d = dg.stereo_bm(_dev(L), _dev(R))
    np.testing.assert_array_equal(d[0].cpu().numpy(), fx["bm"]["shape_288x1280"])
    np.testing.assert_array_equal(d[2].cpu().numpy(), fx["bm"]["shape_288x1280"])
    np.testing.assert_array_equal(d[1].cpu().numpy(), sb.stereo_bm(c["right"], c["left"]))


def _frames(grey, seed):
    """A float32 normalised RGB frame whose channels vary around `grey` (so denorm + BGR2GRAY is not trivial)."""
    rng = np.random.RandomState(seed)
    rgb = np.clip(grey[..., None].astype(np.int64) + rng.randint(-30, 31, grey.shape + (3,)), 0, 255).astype(np.float64)
    img = ((rgb / 255.0 - dc.MEAN) / dc.STD).astype(np.float32)
    img[:4, :8] = 9.0                                            # clipped above 1
    img[4:8, :8] = -9.0                                          # clipped below 0
    return img


@pytest.mark.parametrize("cid", ["bands_0_1_37_190_191", "shape_288x1280", "min_26x217"])
def test_front_end_from_float_frames(cid):
    cv2 = pytest.importorskip("cv2")
    from visualdet3d_b200 import disparity_gt as dg
    c = CASES[cid]
    L = np.stack([_frames(c["left"], 1), _frames(c["left"], 3)])
    R = np.stack([_frames(c["right"], 2), _frames(c["right"], 4)])
    disp, grey = dg.bm_disparity(_dev(L), _dev(R), dc.MEAN, dc.STD, return_grey=True)
    maps = dg.bm_targets(_dev(L), _dev(R), dc.MEAN, dc.STD).cpu().numpy()
    grey = grey.cpu().numpy()
    m = cv2.StereoBM_create(192, 25)
    for b in range(2):
        gl = cv2.cvtColor(sb.denorm(L[b], dc.MEAN, dc.STD), cv2.COLOR_BGR2GRAY)
        gr = cv2.cvtColor(sb.denorm(R[b], dc.MEAN, dc.STD), cv2.COLOR_BGR2GRAY)
        np.testing.assert_array_equal(grey[0, b], gl)
        np.testing.assert_array_equal(grey[1, b], gr)
        ref = m.compute(gl, gr)
        np.testing.assert_array_equal(disp[b].cpu().numpy(), ref)
        ref[ref < 0] = 0
        np.testing.assert_array_equal(maps[b], sb.block_max(ref.astype(np.uint16)))


@pytest.mark.parametrize("case", dc.velo_cases(), ids=lambda c: c["id"])
def test_velo_equals_golden(case, fx):
    from visualdet3d_b200 import disparity_gt as dg
    args = (case["R0_rect"], case["Tr_velo_to_cam"], case["P2"], case["baseline"], case["H"], case["W"])
    full = dg.velo_disparity(_dev(case["points"]), *args).cpu().numpy()
    red = dg.velo_targets(_dev(case["points"]), *args).cpu().numpy()
    ref = fx["velo"][case["id"]]
    np.testing.assert_array_equal(full, dg.velo_disparity_host(case["points"], *args))
    if case["margin"]:
        np.testing.assert_array_equal(full, ref)
        np.testing.assert_array_equal(red, fx["velor"][case["id"]])
    else:
        # BLAS may order the reference's 4x4 products differently: a mismatch needs a point within the margin of a boundary
        bad = np.argwhere(full != ref)
        u, v, _, ok = dc.project(case["points"])
        near = dc.near_boundary(case["points"]) & ok
        hit = {(int(y), int(x)) for x, y in zip(u[near], v[near])}
        assert all((int(y), int(x)) in hit for y, x in bad)
        np.testing.assert_array_equal(red, dg.block_max_host(full))


def test_graph_replay():
    from visualdet3d_b200 import disparity_gt as dg
    c = CASES["shape_97x451"]
    L, R = _dev(c["left"][None]).repeat(2, 1, 1), _dev(c["right"][None]).repeat(2, 1, 1)
    ref = dg.stereo_bm(L, R)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        dg.stereo_bm(L, R)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = dg.stereo_bm(L, R)
    out.fill_(0)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, ref)


def test_bad_inputs_raise():
    from visualdet3d_b200 import disparity_gt as dg
    u8 = torch.zeros((1, 40, 300), dtype=torch.uint8, device="cuda")
    with pytest.raises(ValueError):
        dg.stereo_bm(u8.cpu(), u8.cpu())
    with pytest.raises(TypeError):
        dg.stereo_bm(u8.float(), u8.float())
    with pytest.raises(ValueError):
        dg.stereo_bm(u8, u8[:, :, :299])
    with pytest.raises(ValueError):
        dg.stereo_bm(u8[:, :25], u8[:, :25])
    with pytest.raises(ValueError):
        dg.stereo_bm(u8[:, :, :215], u8[:, :, :215])
    f = torch.zeros((1, 40, 300, 3), device="cuda")
    with pytest.raises(ValueError):
        dg.bm_targets(f, f[..., :2], dc.MEAN, dc.STD)
    with pytest.raises(ValueError):
        dg.bm_targets(f, f, dc.MEAN[:2], dc.STD)
    with pytest.raises(TypeError):
        dg.block_max(torch.zeros((1, 8, 8), dtype=torch.int32, device="cuda"))
    pts = torch.zeros((10, 4), device="cuda")
    with pytest.raises(ValueError):
        dg.velo_disparity(pts.cpu(), dc.R0, dc.TR, dc.P2, 0.54, 288, 1280)
    with pytest.raises(TypeError):
        dg.velo_disparity(pts.double(), dc.R0, dc.TR, dc.P2, 0.54, 288, 1280)
    with pytest.raises(ValueError):
        dg.velo_disparity(pts[:, :2], dc.R0, dc.TR, dc.P2, 0.54, 288, 1280)
    with pytest.raises(ValueError):
        dg.velo_disparity(pts, dc.R0[:3, :3], dc.TR, dc.P2, 0.54, 288, 1280)


CLI = """import os, runpy, sys
ROOT = sys.argv[1]
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle")]
import refload
from visualdet3d_b200.ops import dcn, iou3d
refload.load_reference(device="cuda", dcn_ext=dcn, iou3d_ext=iou3d)
sys.argv = ["disparity_precompute"] + sys.argv[2:]
runpy.run_module("visualdet3d_b200.disparity_precompute", run_name="__main__")
"""


@pytest.mark.parametrize("mode,pc", [("tree_bm", "False"), ("tree_velo", "True")])
def test_cli_writes_the_reference_files(mode, pc, fx):
    import cv2
    with tempfile.TemporaryDirectory() as tmp:
        cfg = dc.write_tree(tmp)
        r = subprocess.run([sys.executable, "-c", CLI, ROOT, f"--config={cfg}", f"--use_point_cloud={pc}"], capture_output=True, text=True,
                           cwd=tmp, timeout=600)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
        disp = os.path.join(tmp, "pre", "training", "disp")
        files = sorted(os.listdir(disp))
        assert [f[:-4] for f in files] == sorted(fx[mode])
        for f in files:
            a = cv2.imread(os.path.join(disp, f), -1)
            assert a.dtype == np.uint16
            np.testing.assert_array_equal(a, fx[mode][f[:-4]], err_msg=f)
