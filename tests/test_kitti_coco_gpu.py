"""-m gpu: the COCO-style KITTI AP on the GPU (vd3d_kitti_eval with ten min-overlap rows, through visualdet3d_b200/kitti_eval.py) against
the unmodified reference's stored eval_class curves and get_coco_eval_result text (tests/golden/make_golden_kitti_coco.py); the
official rows unchanged inside a longer row set; and the command line on the fixture files."""
import numpy as np
import pytest

from test_kitti_coco_cpu import CASES, FX, run_cli
from test_kitti_eval_cpu import write_case
from test_kitti_eval_gpu import BEV_TOL
from visualdet3d_b200 import kitti_eval

pytestmark = pytest.mark.gpu


def annos(fx, tmp_path):
    lab, res, split = write_case(fx, str(tmp_path))
    return kitti_eval._read_annos(lab, res, split)


def coco_curves(fx, tmp_path):
    gt, dt = annos(fx, tmp_path)
    classes = [int(c) for c in fx["classes"]]
    mo = kitti_eval.coco_min_overlaps(kitti_eval._coco_overlap_ranges(classes))
    return kitti_eval.do_eval_v3(gt, dt, classes, mo, kitti_eval._compute_aos(dt))


@pytest.mark.parametrize("case", CASES)
def test_coco_curves_match_reference(case, tmp_path):
    fx = FX[case]
    assert float(fx["margin"]) > 2 * BEV_TOL                    # matching decisions cannot flip within the BEV / 3-D tolerance
    out = coco_curves(fx, tmp_path)
    for m in kitti_eval.METRICS:
        assert out[m]["precision"].shape == fx[f"{m}_precision"].shape == (len(fx["classes"]), 3, 10, kitti_eval.N_SAMPLE_PTS)
        assert np.array_equal(out[m]["precision"], fx[f"{m}_precision"]), m
        assert np.array_equal(out[m]["thresholds"], fx[f"{m}_thresholds"]), m
    o, r = out["bbox"]["orientation"], fx["bbox_orientation"]
    assert np.allclose(o, r, rtol=1e-12, atol=0) and np.array_equal(o == 0, r == 0)
    assert (fx["bbox_precision"][:, :, 0] > fx["bbox_precision"][:, :, -1]).any()   # the rows differ


@pytest.mark.parametrize("case", CASES)
def test_coco_text_matches_reference(case, tmp_path):
    fx = FX[case]
    gt, dt = annos(fx, tmp_path)
    classes = [int(c) for c in fx["classes"]]
    texts = [str(t) for t in fx["texts"]]
    assert [kitti_eval.get_coco_eval_result(gt, dt, c) for c in classes] == texts
    assert kitti_eval.get_coco_eval_result(gt, dt, [kitti_eval.CLASS_TO_NAME[c] for c in classes]) == "".join(texts)


@pytest.mark.parametrize("case", CASES)
def test_coco_style_eval_returns_reference_maps(case, tmp_path):
    fx = FX[case]
    gt, dt = annos(fx, tmp_path)
    classes = [int(c) for c in fx["classes"]]
    aos = bool(fx["compute_aos"])
    got = kitti_eval.do_coco_style_eval(gt, dt, classes, kitti_eval._coco_overlap_ranges(classes), aos)
    ref = [kitti_eval.get_mAP_v2(fx[f"{m}_precision"]).mean(-1) for m in kitti_eval.METRICS]
    ref.append(kitti_eval.get_mAP_v2(fx["bbox_orientation"]).mean(-1) if aos else None)
    for g, r in zip(got[:3], ref[:3]):
        assert g.shape == (len(classes), 3) and np.array_equal(g, r)
    assert (got[3] is None) == (not aos)
    if aos:
        assert np.allclose(got[3], ref[3], rtol=1e-12, atol=0)


def test_official_rows_unchanged_in_a_ten_row_call(tmp_path):
    fx = FX["mixed"]
    gt, dt = annos(fx, tmp_path)
    classes = [int(c) for c in fx["classes"]]
    official = kitti_eval.MIN_OVERLAPS[:, :, classes]
    rows = np.concatenate([official, kitti_eval.coco_min_overlaps(kitti_eval._coco_overlap_ranges(classes))[:8]], 0)
    assert rows.shape == (10, 3, len(classes))
    two = kitti_eval.do_eval_v3(gt, dt, classes, official, True)
    ten = kitti_eval.do_eval_v3(gt, dt, classes, rows, True)
    for m in kitti_eval.METRICS:
        for k in ("precision", "thresholds", "orientation"):
            assert np.array_equal(ten[m][k][:, :, :2], two[m][k], equal_nan=True), (m, k)
    single = kitti_eval.do_eval_v3(gt, dt, classes, rows[9:], True)     # one row
    for m in kitti_eval.METRICS:
        assert np.array_equal(single[m]["precision"], ten[m]["precision"][:, :, 9:], equal_nan=True), m


def test_two_coco_runs_are_identical(tmp_path):
    a = coco_curves(FX["mixed"], tmp_path / "a")
    b = coco_curves(FX["mixed"], tmp_path / "b")
    for m in kitti_eval.METRICS:
        for k in ("precision", "thresholds", "orientation"):
            assert np.array_equal(a[m][k], b[m][k], equal_nan=True), (m, k)


@pytest.mark.parametrize("case", CASES)
def test_cli_prints_official_then_coco_text(case, tmp_path):
    fx = FX[case]
    lab, res, split = write_case(fx, str(tmp_path))
    classes = [int(c) for c in fx["classes"]]
    official = "".join(t + "\n" for t in kitti_eval.evaluate(lab, res, split, classes, gpu=0))
    common = ["--label_path", lab, "--result_path", res, "--label_split_file", split]
    r = run_cli(*common, "--current_classes", ",".join(str(c) for c in classes))
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout == official
    names = ",".join(kitti_eval.CLASS_TO_NAME[c] for c in classes)
    r = run_cli(*common, "--current_classes", names, "--coco", "--gpu", "0")
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout == official + "".join(str(t) + "\n" for t in fx["texts"])

