"""The cost-volume restatements and constructed cases of tests/cost_volume_cases.py, checked without a GPU:
  * psm_cosine64 equals oracle/torch_port.py psm_cosine, and concat_conv3d64 equals torch_port.concat_volume + F.conv3d, on every case;
  * every tag case is exact in fp32 (integer partial sums below 2^24, an exact fp16 split);
  * every perturbation of the restatements changes the expected output of every case it targets, at the stated minimum number of elements:
    a kernel that made that error would fail the GPU test's bit-exact comparison.
"""
import pytest
import torch
import torch.nn.functional as F

import cost_volume_cases as cv
import torch_port as tp

PSM_CASES = cv.TC_CASES + cv.SIMT_CASES + cv.VARIANT_CASES + cv.NCHW_CASES
ids = lambda cases: [c["id"] for c in cases]  # noqa: E731
nchw = lambda x: x.permute(0, 3, 1, 2)  # noqa: E731
MIN_CHANGED = 0.05


def _changed(a, b):
    return int((a != b).sum())


def _valid(B, H, W, D):
    """[B, H, W, D] mask of the elements the reference defines (w >= d)."""
    w = torch.arange(W).reshape(1, 1, W, 1)
    d = torch.arange(D).reshape(1, 1, 1, D)
    return (w >= d).expand(B, H, W, D)


@pytest.mark.parametrize("case", PSM_CASES, ids=ids(PSM_CASES))
def test_psm_restatement_matches_torch_port(case):
    B, H, W, C, D = case["B"], case["H"], case["W"], case["C"], case["D"]
    for L, R in (cv.random_features(B, H, W, C, cv.case_seed(case)), cv.tag_features(B, H, W, C, cv.case_seed(case))):
        want, S = cv.psm_cosine64(L, R, D)
        port = tp.psm_cosine(nchw(L), nchw(R), D, 1).permute(0, 2, 3, 1)
        assert float(((port.double() - want).abs() - cv.simt_bound(C, S)).max()) <= 0.0
        assert bool((want.abs() <= S).all())
        assert bool((want[~_valid(B, H, W, D)] == 0).all())


@pytest.mark.parametrize("case", PSM_CASES, ids=ids(PSM_CASES))
def test_psm_tag_cases_are_exact_in_fp32(case):
    B, H, W, C, D = case["B"], case["H"], case["W"], case["C"], case["D"]
    L, R = cv.tag_features(B, H, W, C, cv.case_seed(case))        # asserts the exact hi / lo split
    want, _ = cv.psm_cosine64(L, R, D)
    sums = want * C
    assert torch.equal(sums, sums.round()) and float(sums.max()) < 2 ** 24
    # the fp32 sum in two different orders and the kernels' two scales (fp32 reciprocal, division) reproduce the restatement exactly
    got, got_div = torch.zeros(B, H, W, D), torch.zeros(B, H, W, D)
    for d in range(min(D, W)):
        prod = L[:, :, d:] * R[:, :, :W - d]
        s_fwd = prod.sum(-1)
        s_rev = prod.flip(-1).cumsum(-1)[..., -1]
        assert torch.equal(s_fwd, s_rev)
        got[:, :, d:, d] = s_fwd * torch.tensor(1.0 / C, dtype=torch.float32)
        got_div[:, :, d:, d] = s_fwd / torch.full_like(s_fwd, C)          # IEEE division, as the generic / NCHW kernels
    assert torch.equal(got, cv.device_scale(want, C)) and torch.equal(got_div, cv.device_scale(want, C, divide=True))
    if C & (C - 1) == 0:
        assert torch.equal(cv.device_scale(want, C).double(), want)


def _psm_perturbations(case):
    """(name, perturbed expectation, elements the error touches, the minimum that must change)."""
    B, H, W, C, D = case["B"], case["H"], case["W"], case["C"], case["D"]
    L, R = cv.tag_features(B, H, W, C, cv.case_seed(case))
    want, _ = cv.psm_cosine64(L, R, D)
    valid = _valid(B, H, W, D)
    w = torch.arange(W).reshape(1, 1, W, 1)
    d = torch.arange(D).reshape(1, 1, 1, D)
    diag = (w == d).expand(B, H, W, D)
    out = []
    for s in (-1, 1):
        # every defined element reads R at w - d + s; the columns whose shifted pixel leaves the row turn 0 (also a change)
        out.append((f"r_shift{s:+d}", cv.psm_cosine64(L, R, D, r_shift=s)[0], valid, 0.9))
    # w == d turns 0, w > d reads the next disparity's pixel
    out.append(("d_shift+1", cv.psm_cosine64(L, R, D, d_shift=1)[0], valid, 0.9))
    out.append(("strict_mask", cv.psm_cosine64(L, R, D, strict=True)[0], diag & valid, 1.0))
    ntiles = B * H * W // cv.TC_TILE
    if ntiles >= 2:
        touched = torch.zeros(B * H * W, D, dtype=torch.bool)
        touched[:2 * cv.TC_TILE] = True
        out.append(("swap_tiles", cv.swap_tiles(want, 0, 1), touched.reshape(B, H, W, D) & valid, 0.9))
    if B >= 2:
        touched = torch.zeros(B, H, W, D, dtype=torch.bool)
        touched[:2] = True
        out.append(("swap_images", cv.psm_cosine64(L, cv.swap_images(R, 0, 1), D)[0], touched & valid, 0.9))
    return want, out


@pytest.mark.parametrize("case", PSM_CASES, ids=ids(PSM_CASES))
def test_psm_perturbations_change_the_tag_expectation(case):
    """Minimum changed elements: all of the w == d column for the strict mask (the tag sums are >= C > 0 there), at least 90% of the touched
    elements for the others (the defined elements; for a tile or image swap those of the two tiles / images).  The least measured on these
    cases is 98.7%: a few tag products collide."""
    want, perturbations = _psm_perturbations(case)
    assert perturbations
    for name, got, touched, frac in perturbations:
        n = int(touched.sum())
        changed = int(((got != want) & touched).sum())
        assert n > 0 and changed >= frac * n, (name, changed, n)


# ---- concat volume + Conv3d pair ----------------------------------------------------------------------------------------------------------
def _cv_operands(case, tag):
    make = cv.tag_conv_operands if tag else cv.random_conv_operands
    return make(case["B"], case["H"], case["W"], case["F"], cv.case_seed(case, 1 if tag else 0))


@pytest.mark.parametrize("case", cv.CONCAT_CASES, ids=ids(cv.CONCAT_CASES))
def test_concat_restatement_matches_torch_port(case):
    B, H, W, D = case["B"], case["H"], case["W"], case["D"]
    for tag in (False, True):
        lf, rf, w1, b1, w2, b2 = _cv_operands(case, tag)
        vol = tp.concat_volume(nchw(lf), nchw(rf), D)
        assert torch.equal(vol.double(), cv.concat_volume64(lf, rf, D))
        r = cv.concat_conv3d64(lf, rf, w1, b1, w2, b2, D)
        want = F.relu(F.conv3d(F.relu(F.conv3d(vol.double(), w1.double(), b1.double(), padding=1)), w2.double(), b2.double(), padding=1))
        assert float((cv.to_device_layout(want) - r["out"]).abs().max()) <= 1e-12 * (1.0 + r["abs_max"])
        # fp32 with PyTorch's own summation order stays inside the bound the device is held to
        f32 = F.relu(F.conv3d(F.relu(F.conv3d(vol, w1, b1, padding=1)), w2, b2, padding=1))
        assert bool(((cv.to_device_layout(f32).double() - r["out"]).abs() <= r["bound"]).all())
        if tag:
            assert r["abs_max"] < 2 ** 24
            assert torch.equal(cv.to_device_layout(f32).double(), r["out"])          # exact in fp32, both ReLUs included
            assert bool((r["mid"] == 0).any()) and bool((r["mid"] > 0).any())        # the first ReLU clips
            assert bool((r["out"] == 0).any()) and bool((r["out"] > 0).any())        # and so does the second


@pytest.mark.parametrize("case", cv.CONCAT_CASES, ids=ids(cv.CONCAT_CASES))
def test_concat_perturbations_change_the_tag_expectation(case):
    """Each error changes at least MIN_CHANGED = 5% of the output elements of the tag case (a strict mask reaches only the columns next to
    w == d, at least 6.5% on these cases; a shifted R feature or disparity every column, at least 14%; a swap of images both images)."""
    B, H, W, D = case["B"], case["H"], case["W"], case["D"]
    lf, rf, w1, b1, w2, b2 = _cv_operands(case, True)
    want = cv.concat_conv3d64(lf, rf, w1, b1, w2, b2, D)["out"]
    checks = [("r_shift-1", dict(r_shift=-1)), ("r_shift+1", dict(r_shift=1)), ("strict_mask", dict(strict=True))]
    if D > 1:
        checks.append(("d_shift+1", dict(d_shift=1)))
    n = want.numel()
    for name, kw in checks:
        got = cv.concat_conv3d64(lf, rf, w1, b1, w2, b2, D, **kw)["out"]
        # at W = 1 only disparity 0 holds data and a shifted R reads outside the row, which zeroes the plane
        assert _changed(got, want) >= MIN_CHANGED * n, (name, _changed(got, want), n)
    if B >= 2:
        got = cv.concat_conv3d64(lf, cv.swap_images(rf, 0, 1), w1, b1, w2, b2, D)["out"]
        assert _changed(got[:2], want[:2]) >= MIN_CHANGED * want[:2].numel()

