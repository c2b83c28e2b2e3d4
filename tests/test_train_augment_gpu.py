"""Training-time augmentation kernel (`vd3d_train_augment`, visualdet3d_b200/train_augment.py:augment_batch) against its host form on the
same descriptors: both chains, frames of the three KITTI sizes in one batch, both cameras of a stereo batch in one launch, mirrored and
swapped samples.  Both forms run the same routine with every product and sum rounded separately, so the bound is 1e-6 and the measured
difference is reported."""
import os
import sys
import types

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT

sys.path.insert(0, os.path.join(ROOT, "tests"))
import train_augment_cases as cases  # noqa: E402
from visualdet3d_b200 import _lib  # noqa: E402
from visualdet3d_b200 import train_augment as ta  # noqa: E402

pytestmark = pytest.mark.gpu


def _batch(name, seeds):
    """The DeferredFrames of one collated batch: all left images, then all right images for the stereo list."""
    aug_list, stereo = cases.LISTS[name]
    aug = ta.TrainAugmentation(aug_list)
    lefts, rights, mirrors = [], [], set()
    for i, seed in enumerate(seeds):
        H, W = cases.SIZES[i % 3]
        left, right = cases.frame(seed, H, W), cases.frame(seed + 1, H, W)
        np.random.seed(seed)
        if stereo:
            lo, ro, *_ = aug(left, right, cases.P2.copy(), cases.P3.copy(), cases.labels(seed, H, W, types.SimpleNamespace))
            assert (lo.frame is right) == bool(lo.mirror)                 # the mirror exchanges the cameras
            rights.append(ro)
        else:
            lo, *_ = aug(left, p2=cases.P2.copy(), labels=cases.labels(seed, H, W, types.SimpleNamespace))
        lefts.append(lo)
        mirrors.add(lo.mirror)
    assert mirrors == {0, 1}
    return lefts + rights


@pytest.mark.parametrize("name", cases.NAMES)
def test_kernel_matches_host_form(name):
    fx = np.load(os.path.join(GOLDEN, "train_augment.npz"))            # the fixture's seeds take both mirror outcomes
    frames = _batch(name, [int(fx[f"{name}_{i}_meta"][0]) for i in range(int(fx[f"{name}_cases"]))])
    _lib.launch_count_reset()
    out = ta.augment_batch(frames, "cuda")
    torch.cuda.synchronize()
    assert _lib.launch_count() == 1                                   # one launch per batch, both cameras included
    got = out.cpu().numpy()
    worst = 0.0
    for i, f in enumerate(frames):
        worst = max(worst, float(np.abs(got[i] - ta.augment_host(f)).max()))
    print(f"{name}: kernel vs host form max |diff| {worst:.2e} over {len(frames)} images")
    assert worst <= 1e-6
    again = ta.augment_batch(frames, "cuda")
    assert torch.equal(out, again)                                    # deterministic: same bits on a second launch


def test_pad_lands_on_the_left_when_mirrored():
    aug_list, _ = cases.LISTS["yolo3d"]
    aug = ta.TrainAugmentation(aug_list[:1] + aug_list[2:])          # no photometric program: the pad is exactly Normalize(0)
    outs = []
    # 270 rows -> 288: 1306 columns, cropped to 1280;  250 rows -> 288: 1037 columns, zero padded to 1280
    for frame in (cases.frame(5, 370, 1224), cases.frame(6, 350, 900)):
        for m in (0, 1):
            np.random.seed(0)
            f = aug(frame, p2=cases.P2.copy(), labels=[])[0]
            f.mirror = m
            outs.append(f)
    got = ta.augment_batch(outs, "cuda").cpu().numpy()
    pad = ((0 - np.array(cases.MEAN, np.float32)) / np.array(cases.STD, np.float32)).astype(np.float32)
    Wr = int(np.round(900 * 288 / 250))
    assert Wr < 1280
    assert np.array_equal(got[2][:, :, Wr:], np.broadcast_to(pad[:, None, None], (3, 288, 1280 - Wr)))
    assert np.array_equal(got[3][:, :, :1280 - Wr], np.broadcast_to(pad[:, None, None], (3, 288, 1280 - Wr)))
    assert np.array_equal(got[3], got[2][:, :, ::-1])
    assert np.array_equal(got[1], got[0][:, :, ::-1])


def test_kernel_tails_match_host_form():
    """An output size that is not a multiple of the 128 x 4 tile (290 x 1250): the partial last column block and row block."""
    frames = []
    for name in ("stereo3d", "yolo3d"):
        aug_list = [dict(c, keywords=dict(c["keywords"], size=(290, 1250))) if c["type_name"] == "Resize" else c for c in cases.LISTS[name][0]]
        aug = ta.TrainAugmentation(aug_list)
        for i, (H, W) in enumerate(cases.SIZES):
            np.random.seed(i)
            frames.append(aug(cases.frame(i, H, W), p2=cases.P2.copy(), labels=[])[0])
    assert {f.mirror for f in frames} == {0, 1}
    warp = [dict(c, keywords=dict(c["keywords"], output_w=1250, output_h=290)) if c["type_name"] == "RandomWarpAffine" else c
            for c in cases.LISTS["km3d"][0]]
    aug = ta.TrainAugmentation(warp)
    for i, (H, W) in enumerate(cases.SIZES):
        np.random.seed(i)
        frames.append(aug(cases.frame(i, H, W), p2=cases.P2.copy(), labels=[])[0])
    got = ta.augment_batch(frames, "cuda").cpu().numpy()
    assert got.shape == (len(frames), 3, 290, 1250)
    worst = max(float(np.abs(got[i] - ta.augment_host(f)).max()) for i, f in enumerate(frames))
    print(f"290x1250 tails: kernel vs host form max |diff| {worst:.2e}")
    assert worst <= 1e-6


def test_plugin_matches_the_reference_training_input(tmp_path):
    """The reference dataset + collate_fn + training function, with and without plugin.install_train_augmentation_into_reference(),
    from the same seed: the module gets the same annotations / P2 / P3 / disparity, and images within the augmentation's host bound."""
    from loss_harness import run_seam_worker
    out = run_seam_worker("train_augment_plugin.py", str(tmp_path))
    assert len(out) == 4
    for arm, r in out.items():
        assert r["transforms"] == ["Compose", "TrainAugmentation"], arm
        assert r["shapes_equal"] and r["others_equal"] and r["rng_equal"] and r["float_images"], (arm, r)
        assert r["image_max_diff"] < 5e-5, (arm, r)
