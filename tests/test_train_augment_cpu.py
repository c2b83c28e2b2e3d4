"""Training-time augmentation (visualdet3d_b200/train_augment.py + `vd3d_train_augment_host`) against fixtures from the unmodified reference
`Compose` of the five shipped train_augmentation lists (tests/golden/make_golden_train_augment.py): normalised images within 5e-5 (the
test-time path holds 2e-5; the HSV round trip of cv2's SIMD colour conversion differs from its scalar formula by an ulp on a few percent
of pixels), P2 / P3 bit-equal, the kept labels equal, and the global numpy RNG at the same position after the call."""
import ctypes
import os
import sys
import types

import numpy as np
import pytest

from conftest import GOLDEN, ROOT

sys.path.insert(0, os.path.join(ROOT, "tests"))
import train_augment_cases as cases  # noqa: E402
from visualdet3d_b200 import _lib  # noqa: E402
from visualdet3d_b200 import train_augment as ta  # noqa: E402

TOL = 5e-5


def _fixture():
    return np.load(os.path.join(GOLDEN, "train_augment.npz"))


def _run(name, seed, H, W):
    aug_list, stereo = cases.LISTS[name]
    left, right = cases.frame(seed, H, W), cases.frame(seed + 1, H, W)
    objs = cases.labels(seed, H, W, types.SimpleNamespace)
    np.random.seed(seed)
    aug = ta.TrainAugmentation(aug_list)
    if stereo:
        lo, ro, p2, p3, lab = aug(left, right, cases.P2.copy(), cases.P3.copy(), objs)
        imgs = {"l": lo, "r": ro}
    else:
        lo, p2, lab = aug(left, p2=cases.P2.copy(), labels=objs)
        p3 = np.zeros((3, 4))
        imgs = {"l": lo}
    return imgs, p2, p3, lab, np.random.rand()


def _cases(fx):
    for name in cases.NAMES:
        for ci in range(int(fx[f"{name}_cases"])):
            k = f"{name}_{ci}"
            seed, H, W, _ = [int(v) for v in fx[f"{k}_meta"]]
            yield name, k, seed, H, W


def test_host_form_matches_reference_fixtures():
    fx = _fixture()
    worst = 0.0
    for name, k, seed, H, W in _cases(fx):
        imgs, p2, p3, lab, nxt = _run(name, seed, H, W)
        assert nxt == float(fx[f"{k}_next_rand"]), (k, "numpy RNG position differs from the reference's")
        assert np.array_equal(p2, fx[f"{k}_P2"]) and np.array_equal(p3, fx[f"{k}_P3"]), (k, "calibration")
        assert np.array_equal(cases.label_array(lab), fx[f"{k}_labels"]), (k, "labels")
        for side, f in imgs.items():
            assert f.shape == (384 if name in ("monoflex", "km3d") else 288, 1280, 3)
            out = ta.augment_host(f)
            st = int(fx[f"{k}_{side}_stride"])
            d = max(float(np.abs(out.reshape(-1)[::st] - fx[f"{k}_{side}_samples"]).max()),
                    float(np.abs(out[:, 0, :] - fx[f"{k}_{side}_first_row"]).max()),
                    float(np.abs(out[:, :, -1] - fx[f"{k}_{side}_last_col"]).max()))
            worst = max(worst, d)
            assert d < TOL, (k, side, d)
            assert abs(float(out.astype(np.float64).sum()) - float(fx[f"{k}_{side}_sum"])) < 1e-6 * float(fx[f"{k}_{side}_abssum"]), (k, side)
    print(f"train augmentation host form: max |diff| vs the reference {worst:.2e}")


def test_fixture_cases_cover_every_branch():
    fx = _fixture()
    mirrors, orders = {}, {}
    border = set()
    for name, k, seed, H, W in _cases(fx):
        imgs, *_ = _run(name, seed, H, W)
        f = imgs["l"]
        ops = [int(o) for o in f.ops]
        mirrors.setdefault(name, set()).add(f.mirror)
        if name in ("monoflex", "km3d"):
            first = [ops.index(c) for c in (ta.OP_BRIGHTNESS, ta.OP_CONTRAST, ta.OP_RGB2HSV)]
            orders.setdefault(name, set()).add(tuple(np.argsort(first)))
            # the warp centre (inverse map of the output centre) within a few pixels of the randint range's ends
            a = f.affine.astype(np.float64)
            cw, ch = (640 - a[0, 2]) / a[0, 0], (192 - a[1, 2]) / a[1, 1]
            if min(cw - 128, W - 129 - cw) < 24.5 or min(ch - 128, H - 129 - ch) < 8.5:
                border.add(name)
            assert ops.count(ta.OP_EIGEN_NOISE) == (name == "km3d")
        else:
            assert ops[0] == ta.OP_BRIGHTNESS and len(ops) == 6
            orders.setdefault(name, set()).add((f.mirror, ops.index(ta.OP_CONTRAST) < ops.index(ta.OP_RGB2HSV)))
    for name in cases.NAMES:
        assert mirrors[name] == {0, 1}, name
        if name in ("monoflex", "km3d"):
            assert len(orders[name]) == 6, (name, orders[name])
            assert name in border, name
        else:
            assert len(orders[name]) == 4, (name, orders[name])


def _describe(**over):
    a = dict(H=375, W=1242, C=3, geom=0, crop_top=100, Ho=288, Wo=1280, mirror=0, ops=[ta.OP_BRIGHTNESS], args=[3.0],
             affine=np.array([[1.0, 0, 0], [0, 1.0, 0]], np.float32), null_src=False)
    a.update(over)
    frame = np.zeros((a["H"], a["W"], 3), np.uint8)
    desc = np.zeros(int(_lib.load().vd3d_train_augment_desc_bytes()), np.uint8)
    ops, args = np.array(a["ops"], np.int32), np.array(a["args"], np.float32)
    vp = lambda x: x.ctypes.data_as(ctypes.c_void_p)
    src = None if a["null_src"] else frame.ctypes.data
    _lib.call("vd3d_train_augment_describe", vp(desc), src, a["H"], a["W"], a["C"], a["W"] * 3, a["geom"], a["crop_top"],
              a["Ho"], a["Wo"], vp(a["affine"]), a["mirror"], len(ops), vp(ops), vp(args), None)
    return desc


@pytest.mark.parametrize("over, msg", [
    (dict(C=4), "bad arguments"),
    (dict(mirror=2), "bad arguments"),
    (dict(geom=3), "unknown geometry"),
    (dict(ops=[9], args=[0.0]), "unknown op code"),
    (dict(ops=[ta.OP_EIGEN_NOISE], args=[0.0]), "without its vector"),
    (dict(ops=[1] * 9, args=[0.0] * 9), "photometric program"),
    (dict(crop_top=375), "crop_top"),
    (dict(Wo=0), "bad arguments"),
    (dict(H=900, W=3000, crop_top=0, Ho=288), "shrinks"),
    (dict(geom=1, affine=np.zeros((2, 3), np.float32)), "singular"),
    (dict(null_src=True), "bad arguments"),
])
def test_bad_descriptors_are_rejected(over, msg):
    with pytest.raises(_lib.Vd3dError, match=msg):
        _describe(**over)


def test_host_entry_rejects_a_mismatched_output():
    desc = _describe()
    out = np.empty((3, 288, 1000), np.float32)
    m = np.zeros(3, np.float32)
    vp = lambda x: x.ctypes.data_as(ctypes.c_void_p)
    with pytest.raises(_lib.Vd3dError, match="descriptor made for"):
        _lib.call("vd3d_train_augment_host", vp(desc), 3, 288, 1000, vp(m), vp(m + 1), vp(out))
    with pytest.raises(_lib.Vd3dError, match="bad arguments"):
        _lib.call("vd3d_train_augment_host", vp(desc), 4, 288, 1280, vp(m), vp(m + 1), vp(out))


@pytest.mark.parametrize("cfg", [
    {"type_name": "RandomCropToWidth", "keywords": {"width": 1216}},
    {"type_name": "CropTop", "keywords": {"output_height": 352}},
    {"type_name": "ResizeToFx", "keywords": {"Fx": 721.5337}},
    {"type_name": "CropRight", "keywords": {"output_width": 1216}},
    {"type_name": "ConvertColor", "keywords": {"current": "RGB", "transform": "LAB"}},
])
def test_unsupported_transforms_raise_at_construction(cfg):
    aug_list = list(cases.LISTS["stereo3d"][0])
    aug_list.insert(2, cfg)
    name = cfg["type_name"]
    with pytest.raises(NotImplementedError, match=name):
        ta.TrainAugmentation(aug_list)
    assert not ta.supports(aug_list)


def test_unsupported_sequences_raise():
    base = cases.LISTS["stereo3d"][0]
    for bad in (base[1:],                                              # photometric program on the uint8 frame
                base[:-1],                                             # no Normalize
                [base[0], base[2], base[3], base[1], base[4], base[5]],   # program after the resize
                base[:5] + [base[4], base[5]]):                        # two mirrors
        with pytest.raises(NotImplementedError):
            ta.TrainAugmentation(bad)
    for name in cases.NAMES:
        assert ta.supports(cases.LISTS[name][0])
    aug = ta.TrainAugmentation(base)
    img = cases.frame(0, 375, 1242)
    with pytest.raises(NotImplementedError, match="image_gt"):
        aug(img, img, cases.P2.copy(), cases.P3.copy(), [], image_gt=np.zeros((375, 1242), np.float32))
