"""The det_precompute CLI and the anchor-prior accumulation without a GPU: the host entry (the parity checker) against the reference's
own computation on constructed cases, the float32-form bin table, the header-only geometry, and the CLI's host paths against the files
the unmodified reference scripts wrote (tests/golden/det_precompute.npz)."""
import hashlib
import os
import sys
import tempfile

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
import det_precompute_cases as dc

SHA256 = "0a6f276f562d278e3dcbadfca97f2155707acb2edb6d53cbfaefc550d39b6fbb"


@pytest.fixture(scope="module")
def fx():
    z = np.load(os.path.join(GOLDEN, "det_precompute.npz"))
    return {k: z[k] for k in z.files}


def _ref():
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import refload
    if not refload.available():
        pytest.skip("the reference package is not available")
    refload.load_reference()
    sys.path.insert(0, GOLDEN)
    import make_golden_det_precompute as mg
    return mg


def test_fixture_sha():
    with open(os.path.join(GOLDEN, "det_precompute.npz"), "rb") as f:
        assert hashlib.sha256(f.read()).hexdigest() == SHA256


def host_state(c):
    from visualdet3d_b200 import anchor_prior as ap
    st = ap.PriorState(c["T"], c["n_bins"])
    order, start = ap.bin_order(c["bins"], c["n_bins"])
    ap.accumulate_host(st, c["anchors"], order, start, c["offsets"], c["boxes"], c["gt3"], c["thr"])
    return st.numpy()


CASES = {c["id"]: c for c in dc.kernel_cases()}


@pytest.mark.parametrize("cid", sorted(CASES))
def test_host_entry_equals_golden(cid, fx):
    st = host_state(CASES[cid])
    for k in ("examine", "sums", "squared", "usable"):
        np.testing.assert_array_equal(st[k], fx[f"case/{cid}/{k}"], err_msg=f"{cid} {k}")


def _priors(cid, fx):
    from visualdet3d_b200.anchor_prior import priors_from_state
    st = {k: fx[f"case/{cid}/{k}"] for k in ("examine", "sums", "squared", "usable")}
    T = CASES[cid]["T"]
    return priors_from_state(st, CASES[cid]["n_bins"], 1, np.ones((T, 6)), np.ones((T, 6)) * 2, [1] * T)


def test_cases_reach_their_claims(fx):
    g = lambda cid, k: fx[f"case/{cid}/{k}"]
    assert g("iou_exactly_half", "examine").tolist() == [[0, 1]]
    assert g("identical_gts", "sums")[0, 0, 0] == 7.0 and g("identical_gts", "examine")[0, 0] == 1
    assert g("tied_gts", "sums")[0, 0, 0] == 3.0 and g("tied_gts", "examine")[0, 0] == 1
    assert g("zero_area_gt", "usable").tolist() == [1] and g("unreachable_gt", "usable").tolist() == [1]
    assert float(np.float32(0.6)) > 0.6 and g("threshold_f32", "examine")[0, 0] == 0 and g("threshold_f64", "examine")[0, 0] == 0
    assert g("few_positives", "examine")[0, 0] == 9 and _priors("few_positives", fx)[0][0][0, 0, 0] == -100
    assert g("same_z", "examine")[0, 0] == 12 and _priors("same_z", fx)[0][1][0, 0, 0] == 1e10
    ex = float(g("negative_variance", "examine")[0, 0]) + 1e-8
    avg, ex2 = g("negative_variance", "sums")[0, 0, 0] / ex, g("negative_variance", "squared")[0, 0, 0] / ex
    assert ex2 - avg ** 2 < 0 and _priors("negative_variance", fx)[0][0][0, 0, 0] == -100
    # the float64 path: each case's outcome flips under the other rule
    assert g("f64_threshold_flip", "examine")[0, 0] == 1 and g("f64_threshold_flip", "usable")[0] == 1
    assert g("f64_threshold_flip_as_f32", "examine")[0, 0] == 0 and g("f64_threshold_flip_as_f32", "usable")[0] == 0
    assert np.float32(10) * np.float32(6.0000001) / np.float32(100) == np.float32(0.6)
    assert g("f64_anchor_area_f32", "examine")[0, 0] == 1 and g("f64_anchor_area_f32", "usable")[0] == 1
    h = dc.AREA_BOX_H
    a32 = float(np.float32(4097) * np.float32(4097))
    assert a32 == dc.ANCHOR_AREA32 != 4097 * 4097

    def iou64(anchor_area):
        inter = 4097.0 * h
        return inter / ((anchor_area + 4097.0 * h) - inter)
    assert iou64(a32) > 0.5 and not iou64(4097.0 * 4097.0) > 0.5
    f, hf = np.float32, np.float32(h)
    assert not (f(4097) * hf) / ((f(a32) + f(4097) * hf) - f(4097) * hf) > f(0.5)
    k = np.diff(CASES["k_edges"]["offsets"])
    assert 0 in k and 512 in k
    for cid in ("many_frames_f32", "many_frames_f64"):
        c = CASES[cid]
        per_bin = np.bincount(c["bins"], minlength=c["n_bins"])
        assert len(c["anchors"]) % 256 and len(c["anchors"]) > 5 * 256 and (per_bin * c["B"]).min() > 1024
        assert (g(cid, "examine") > 0).sum() >= c["n_bins"]
    assert CASES["many_frames_f64"]["boxes"].dtype == np.float64 and CASES["many_frames_f32"]["boxes"].dtype == np.float32


def test_bin_table_equals_anchors2indexes():
    _ref()
    import torch
    from visualDet3D.networks.heads.anchors import Anchors
    from visualdet3d_b200.anchor_prior import bin_table32
    from visualdet3d_b200.anchors import grid_anchors
    for ratios, hw in (([0.5, 1, 2.0], (288, 1280)), ([0.5, 1], (288, 1280)), ([0.5, 1, 2.0], (275, 1242))):
        cfg = dict(pyramid_levels=[4], strides=[16], sizes=[24], ratios=np.array(ratios), scales=np.array([2 ** (i / 4.0) for i in range(16)]))
        ref = Anchors("", readConfigFile=False, **cfg)
        a_ref = ref(torch.zeros((1, 3) + hw))[0].numpy()
        a32 = grid_anchors(hw, *(cfg[k] for k in ("pyramid_levels", "strides", "sizes", "ratios", "scales"))).astype(np.float32)
        np.testing.assert_array_equal(a32, a_ref)
        for mine, theirs in zip(bin_table32(a32, cfg["sizes"], cfg["ratios"], cfg["scales"]), ref.anchors2indexes(a_ref)):
            np.testing.assert_array_equal(mine, theirs)


def test_multilevel_anchor_config_names_the_config():
    from visualdet3d_b200.anchor_prior import AnchorPriorAccumulator
    cfg = dict(pyramid_levels=[3, 4, 5, 6, 7], strides=[8, 16, 32, 64, 128], sizes=[32, 64, 128, 256, 512], ratios=np.array([0.5, 1, 2.0]),
               scales=np.array([2 ** (i / 3.0) for i in range(3)]))
    with pytest.raises(ValueError, match="RetinaNet"):
        AnchorPriorAccumulator(cfg, (288, 1280), ["Car"], 0.5, None, "RetinaNet")


@pytest.mark.parametrize("name", sorted(dc.TEST_LISTS))
def test_header_geometry_equals_the_reference_compose(name):
    _ref()
    import refload
    from copy import deepcopy
    from visualDet3D.data.kitti.kittidata import KittiData, read_image
    from visualDet3D.data.pipeline import build_augmentator
    from visualdet3d_b200.det_precompute import TestGeometry
    aug = eval(dc.TEST_LISTS[name], {"edict": refload.EasyDict, "np": np})
    geo = TestGeometry(aug)
    assert geo.host == (name != "MonoDepth")
    compose = build_augmentator(aug)
    with tempfile.TemporaryDirectory() as tmp:
        raw, _ = dc.write_tree(tmp, n_frames=8)
        for i in range(8):
            kd = KittiData(raw, "%06d" % i, {"calib": True, "image": False, "label": True, "velodyne": False})
            calib, _, label, _ = kd.read_data()
            hw, p2, labels = geo(kd.image2_path, calib.P2, label.data)
            img, p2r, lr = compose(read_image(kd.image2_path), p2=deepcopy(calib.P2), labels=deepcopy(label.data))
            assert tuple(hw) == img.shape[:2]
            np.testing.assert_array_equal(p2, p2r)
            assert len(labels) == len(lr)
            for a, b in zip(labels, lr):
                assert vars(a) == vars(b) and all(type(vars(a)[k]) is type(vars(b)[k]) for k in vars(a))


def _pickles_equal(mg, tmp, prefix, path, fx):
    out = {}
    mg.flatten_pickle(path, tmp, prefix, out)
    for k, v in out.items():
        np.testing.assert_array_equal(v, fx[k], err_msg=k)
    assert sorted(k for k in fx if k.startswith(prefix)) == sorted(out)


def test_host_cli_paths_equal_the_reference(fx):
    """Every config through read_one_split with the state on the host (the parity checker), and --split=test: the reference's files."""
    mg = _ref()
    from visualDet3D.utils.utils import cfg_from_file
    from visualdet3d_b200 import det_precompute as dp
    with tempfile.TemporaryDirectory() as tmp:
        raw, split = dc.write_tree(tmp)
        for name in dc.CONFIGS:
            cfg = cfg_from_file(dc.write_config(name, tmp, raw, split))
            tr, va = dp.process_train_val_file(cfg)
            dp.read_one_split(cfg, tr, raw, {"calib": True, "image": True, "label": True, "velodyne": False}, 'training', 100, device=None)
            dp.read_one_split(cfg, va, raw, {"calib": True, "image": False, "label": True, "velodyne": False}, 'validation', 100, device=None)
            for sp in ("training", "validation"):
                d = os.path.join(cfg.path.preprocessed_path, sp)
                npys = sorted(f[:-4] for f in os.listdir(d) if f.endswith(".npy"))
                assert npys == sorted(k[len(f"{name}/{sp}/"):] for k in fx if k.startswith(f"{name}/{sp}/anchor_"))
                for f in npys:
                    np.testing.assert_array_equal(np.load(os.path.join(d, f + ".npy")), fx[f"{name}/{sp}/{f}"], err_msg=f"{name} {f}")
                _pickles_equal(mg, tmp, f"{name}/{sp}/pkl/", os.path.join(d, "imdb.pkl"), fx)
        cfgp = dc.write_config("stereo3d", tmp, raw, split)
        dp.main(cfgp, "test")
        _pickles_equal(mg, tmp, "test/test/pkl/", os.path.join(cfg_from_file(cfgp).path.preprocessed_path, "test", "imdb.pkl"), fx)


def test_golden_covers_both_iou_paths_and_the_empty_class(fx):
    assert np.isnan(fx["stereo3d_f64/training/anchor_mean_Van"][..., 3:]).all()
    assert not np.isnan(fx["stereo3d/training/anchor_mean_Car"]).any()
    assert (fx["stereo3d/training/anchor_mean_Car"][..., 0] > -100).sum() > 0


def test_cli_arguments():
    from visualdet3d_b200.det_precompute import parse_args
    a = parse_args(["--config=c.py"])
    assert (a.config, a.split) == ("c.py", "train")
    assert parse_args(["--config=c.py", "--split=test"]).split == "test"
    for bad in (["--config=c.txt"], ["--config=c.py", "--split=val"]):
        with pytest.raises(SystemExit):
            parse_args(bad)


def test_accumulator_follows_each_segments_dtype():
    """Each (frame, class) segment takes torch.tensor's dtype of its own values, as in the script: numpy float64 boxes are positive, python
    floats are not, also when one frame or one class mixes the two."""
    from visualdet3d_b200.anchor_prior import AnchorPriorAccumulator, _box_dtype
    import torch
    assert _box_dtype([list(dc.FLIP_BOX)]) == torch.float32
    assert _box_dtype([[np.float64(v) for v in dc.FLIP_BOX]]) == torch.float64
    with pytest.raises(TypeError):
        _box_dtype([[3, 3, 13, 9]])
    acc = AnchorPriorAccumulator(dc.FLIP_CFG, (16, 16), ["Car", "Pedestrian"], 0.6, None)
    acc.add(dc.dtype_frames())
    st = acc.state.numpy()
    assert st["examine"][:, 0].tolist() == [2, 1] and st["usable"].tolist() == [2, 1]


def test_batches_are_capped_by_the_workspace(monkeypatch):
    """A batch larger than the positive-box workspace budget is split into launches; the state is the same bits."""
    from visualdet3d_b200 import anchor_prior as ap
    c = CASES["many_frames_f32"]
    frames = []
    for b in range(c["B"]):
        objs = []
        for t, typ in enumerate(("Car", "Pedestrian")):
            s = b * 2 + t
            for k in range(c["offsets"][s], c["offsets"][s + 1]):
                z, sn, cs = c["gt3"][k]
                objs.append(dc.label(typ, tuple(float(v) for v in c["boxes"][k]), z=float(z), alpha=float(np.arctan2(sn, cs) / 2)))
        frames.append(objs)
    cfg = dict(pyramid_levels=[4], strides=[16], sizes=[24], ratios=np.array([0.5, 1.0, 2.0]), scales=np.array([1.0, 2 ** 0.5, 2.0, 2 ** 1.5]))
    whole = ap.AnchorPriorAccumulator(cfg, (96, 320), ["Car", "Pedestrian"], 0.5, None)
    whole.add(frames)
    monkeypatch.setattr(ap, "MAX_FLAG_BYTES", 4 * 1440 * 2 * 3)          # three frames per launch
    assert ap.max_frames_per_launch(1440, 2) == 3
    split = ap.AnchorPriorAccumulator(cfg, (96, 320), ["Car", "Pedestrian"], 0.5, None)
    split.add(frames)
    for k, v in whole.state.numpy().items():
        assert v.tobytes() == split.state.numpy()[k].tobytes(), k
    assert whole.state.numpy()["examine"].sum() > 0
    assert ap.max_frames_per_launch(69120, 2) * 2 * 69120 * 4 <= (1 << 30)


@pytest.mark.parametrize("step", ["resize_stretch", "croptop_by_height"])
def test_geometry_without_a_host_form_falls_back(step):
    _ref()
    import refload
    from visualdet3d_b200.det_precompute import TestGeometry
    E = refload.EasyDict
    s = E(type_name="Resize", keywords=E(size=(288, 1280), preserve_aspect_ratio=False)) if step == "resize_stretch" else \
        E(type_name="CropTop", keywords=E(output_height=300))
    geo = TestGeometry([E(type_name="ConvertToFloat"), s])
    assert not geo.host
    with tempfile.TemporaryDirectory() as tmp:
        raw, _ = dc.write_tree(tmp, n_frames=1)
        from visualDet3D.data.kitti.kittidata import KittiData
        kd = KittiData(raw, "000000", {"calib": True, "image": False, "label": True, "velodyne": False})
        calib, _, label, _ = kd.read_data()
        hw, _, _ = geo(kd.image2_path, calib.P2, label.data)
        assert tuple(hw) == ((288, 1280) if step == "resize_stretch" else (300, 1242))
