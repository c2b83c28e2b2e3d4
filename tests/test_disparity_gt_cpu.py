"""CPU checks of Stereo3D's disparity ground truth (csrc/disparity_gt.cu host entries, oracle/stereo_bm.py, the precompute CLI's
arguments) against tests/golden/disparity_gt.npz (cv2 4.13 and the unmodified reference; tests/golden/make_golden_disparity_gt.py)."""
import hashlib
import os

import numpy as np
import pytest

from conftest import GOLDEN, load_fixture
import disparity_gt_cases as dc
import stereo_bm as sb

FIXTURE_SHA256 = "1d12a36300b6d18560e9bf35583f800b7e99c32c0eb46948608373af25dc1255"
CASES = {c["id"]: c for c in dc.bm_cases()}
SMALL = [k for k, c in CASES.items() if c["left"].size <= 200 * 480]


@pytest.fixture(scope="module")
def fx():
    return load_fixture("disparity_gt")


def test_fixture_sha():
    with open(os.path.join(GOLDEN, "disparity_gt.npz"), "rb") as f:
        assert hashlib.sha256(f.read()).hexdigest() == FIXTURE_SHA256


@pytest.mark.parametrize("cid", list(CASES))
def test_oracle_equals_cv2_and_golden(cid, fx):
    c = CASES[cid]
    mine = sb.stereo_bm(c["left"], c["right"])
    np.testing.assert_array_equal(mine, fx["bm"][cid])
    cv2 = pytest.importorskip("cv2")
    np.testing.assert_array_equal(mine, cv2.StereoBM_create(192, 25).compute(c["left"], c["right"]))
    np.testing.assert_array_equal(sb.block_max(mine), fx["bmr"][cid])


@pytest.mark.parametrize("cid", SMALL)
def test_case_reaches_its_claims(cid, fx):
    c = CASES[cid]
    H, W = c["left"].shape
    C, T = sb.cost_volume(c["left"], c["right"])
    out, m = fx["bm"][cid], sb.valid_mask(H, W)
    mn = C.min(0)
    frac = (out.astype(int) + 8) % 16 - 8
    for claim in c["claims"]:
        if claim == "bands":
            for r0, r1, d in dc.interior(c):
                # columns 0 and W-1 are 31 in both frames, which the shifted texture does not match: windows reaching them are left out
                blk = out[r0:r1, sb.X0 + 1:W - 13]
                assert (C[sb.ND - 1 - d, r0:r1, sb.X0 + 1:W - 13] == 0).all()
                assert (np.abs(blk.astype(int) - 16 * d) <= 8).all()
                if d in (0, 191):                    # the sad[-1] / sad[ND] mirror: p == n, so no sub-pixel step
                    assert (blk == 16 * d).all()
        elif claim == "subpixel":
            assert ((frac > 0) & (out > 0) & m).any() and ((frac < 0) & (out > 0) & m).any()
        elif claim == "texture":
            assert ((T < sb.TEXTURE) & m).any() and (out[(T < sb.TEXTURE) & m] == sb.FILTERED).all()
        elif claim == "unique":
            assert ((T >= sb.TEXTURE) & m & (out == sb.FILTERED)).any()
        elif claim == "tie":
            tie = np.zeros((H, W), bool)
            for k in range(sb.ND - 1):
                tie |= (C[k] == mn) & (C[k + 1] == mn) & (np.argmin(C, 0) == k)
            assert (tie & m & (out > sb.FILTERED)).any()
        elif claim == "saturate":
            P = sb.prefilter(c["left"])
            assert P.min() == 0 and P.max() == 2 * sb.CAP
        elif claim == "defined":
            assert (out[m] > sb.FILTERED).any()


@pytest.mark.parametrize("cid", [k for k in CASES if k not in SMALL])
def test_large_cases_hold_their_bands(cid, fx):
    c = CASES[cid]
    out = fx["bm"][cid]
    for r0, r1, d in dc.interior(c):
        assert (np.abs(out[r0:r1, sb.X0 + 1:c["left"].shape[1] - 13].astype(int) - 16 * d) <= 8).all()


def test_grey_formula_equals_cv2():
    cv2 = pytest.importorskip("cv2")
    img = np.random.RandomState(0).randint(0, 256, (512, 512, 3)).astype(np.uint8)
    np.testing.assert_array_equal(sb.grey(img), cv2.cvtColor(img, cv2.COLOR_BGR2GRAY))


def test_host_grey_equals_denorm_and_cvtcolor():
    cv2 = pytest.importorskip("cv2")
    from visualdet3d_b200 import disparity_gt as dg
    rng = np.random.RandomState(1)
    img = (rng.randn(96, 128, 3) * 1.5).astype(np.float32)
    img[10:20] = ((np.array([100, 150, 200]) / 255.0 - dc.MEAN) / dc.STD).astype(np.float32)       # flat region at exact levels
    np.testing.assert_array_equal(dg.grey_host(img, dc.MEAN, dc.STD), cv2.cvtColor(sb.denorm(img, dc.MEAN, dc.STD), cv2.COLOR_BGR2GRAY))


@pytest.mark.parametrize("cid", list(CASES))
def test_host_entry_equals_golden(cid, fx):
    from visualdet3d_b200 import disparity_gt as dg
    c = CASES[cid]
    d = dg.stereo_bm_host(c["left"], c["right"])
    np.testing.assert_array_equal(d, fx["bm"][cid])
    np.testing.assert_array_equal(dg.block_max_host(d), fx["bmr"][cid])


@pytest.mark.parametrize("case", dc.velo_cases(), ids=lambda c: c["id"])
def test_host_velo_equals_golden(case, fx):
    from visualdet3d_b200 import disparity_gt as dg
    ref = fx["velo"][case["id"]]
    mine = dg.velo_disparity_host(case["points"], case["R0_rect"], case["Tr_velo_to_cam"], case["P2"], case["baseline"], case["H"],
                                  case["W"])
    if case["margin"]:
        np.testing.assert_array_equal(mine, ref)
    else:
        bad = np.argwhere(mine != ref)
        u, v, _, ok = dc.project(case["points"])
        near = dc.near_boundary(case["points"])
        hit = {(int(y), int(x)) for x, y in zip(u[near & ok], v[near & ok])} if bad.size else set()
        assert all((int(y), int(x)) in hit for y, x in bad), f"{len(bad)} pixels differ without a point near a boundary"
    assert (mine > 0).sum() > 1000
    np.testing.assert_array_equal(dg.block_max_host(mine), fx["velor"][case["id"]])


def test_velo_cases_reach_their_claims():
    c = dc.velo_cases()
    margin, scan = c[0]["points"], c[1]["points"]
    assert not dc.near_boundary(margin).any()
    u, v, z, ok = dc.project(margin)
    pix = np.stack([v[ok].astype(int), u[ok].astype(int)], 1)
    _, counts = np.unique(pix, axis=0, return_counts=True)
    assert (counts >= 2).sum() >= 1000                          # several points per pixel
    assert (~ok & (margin[:, 0] > 2)).sum() >= 500 and (margin[:, 0] <= 2).sum() >= 500
    assert 100000 <= len(scan) and dc.project(scan)[3].sum() > 5000


def test_host_rejects_undefined_shapes():
    from visualdet3d_b200 import disparity_gt as dg
    a = np.zeros((25, 300), np.uint8)
    with pytest.raises(ValueError):
        dg.stereo_bm_host(a, a)
    a = np.zeros((40, 215), np.uint8)
    with pytest.raises(ValueError):
        dg.stereo_bm_host(a, a)
    with pytest.raises(ValueError):
        sb.stereo_bm(a, a)


def test_cli_arguments():
    from visualdet3d_b200.disparity_precompute import parse_args
    a = parse_args(["--config=cfg/x.py", "--use_point_cloud=True"])
    assert a.config == "cfg/x.py" and a.use_point_cloud is True
    assert parse_args(["--config=x.py", "--use_point_cloud=False"]).use_point_cloud is False
    assert parse_args(["--config=x.py"]).use_point_cloud is False
    assert parse_args(["--config=x.py", "--use_point_cloud"]).use_point_cloud is True
    for bad in (["--config=x.py", "--use_point_cloud=maybe"], ["--config=x.txt"], ["--nonsense"]):
        with pytest.raises(SystemExit):
            parse_args(bad)
