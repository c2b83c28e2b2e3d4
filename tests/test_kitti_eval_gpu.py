"""The native KITTI evaluator on the GPU (csrc/kitti_eval.cu through visualdet3d_b200/kitti_eval.py) against the unmodified reference
evaluator's outputs (tests/golden/make_golden_kitti_eval.py): rotated IoU, per-image overlaps, precision / thresholds / orientation of
every metric, and the text `evaluate()` returns."""
import numpy as np
import pytest
import torch

from test_kitti_eval_cpu import CASES, FX, write_case
from visualdet3d_b200 import kitti_eval

pytestmark = pytest.mark.gpu
BEV_TOL = 1e-5     # float32 BEV / 3-D overlaps: the reference's come from the numba CUDA simulator, which rounds differently


@pytest.mark.parametrize("criterion", [-1, 0, 1, 2])
def test_rotate_iou_matches_reference(criterion):
    fx = FX["riou"]
    got = kitti_eval.rotate_iou(torch.from_numpy(fx["boxes"]).cuda(), torch.from_numpy(fx["qboxes"]).cuda(), criterion).cpu().numpy()
    ref = fx[f"crit{criterion}"]
    assert got.shape == ref.shape and got.dtype == np.float32
    assert (ref > 0).mean() > 0.3                               # the fixture overlaps
    assert np.abs(got.astype(np.float64) - ref).max() < BEV_TOL


def run_case(fx, tmp_path):
    lab, res, split = write_case(fx, str(tmp_path))
    gt = kitti_eval.get_label_annos(lab, kitti_eval._read_imageset_file(split))
    dt = kitti_eval.get_label_annos(res)
    classes = [int(c) for c in fx["classes"]]
    compute_aos = kitti_eval._compute_aos(dt)
    return kitti_eval.do_eval_v3(gt, dt, classes, kitti_eval.MIN_OVERLAPS[:, :, classes], compute_aos, return_overlaps=True)


@pytest.mark.parametrize("case", CASES)
def test_overlaps_and_curves_match_reference(case, tmp_path):
    fx = FX[case]
    assert float(fx["margin"]) > 2 * BEV_TOL                    # matching decisions cannot flip within the BEV / 3-D tolerance
    out = run_case(fx, tmp_path)
    got = np.concatenate([o.reshape(3, -1) for o in out["overlaps"]], 1)
    ref = fx["overlaps"]
    assert got.shape == ref.shape
    assert np.array_equal(got[0], ref[0])                      # bbox: float64 in the reference's order, bit-identical
    assert np.abs(got[1:] - ref[1:]).max() < BEV_TOL
    for m in kitti_eval.METRICS:
        assert np.array_equal(out[m]["precision"], fx[f"{m}_precision"]), m
        assert np.array_equal(out[m]["thresholds"], fx[f"{m}_thresholds"]), m
    o, r = out["bbox"]["orientation"], fx["bbox_orientation"]
    assert np.allclose(o, r, rtol=1e-12, atol=0) and np.array_equal(o == 0, r == 0)
    assert (fx["bbox_thresholds"] > 0).any()
    assert (fx["3d_precision"] > 0).any() == (case != "bbox2d")    # 2-D results carry placeholder 3-D boxes


@pytest.mark.parametrize("case", CASES)
def test_evaluate_returns_reference_text(case, tmp_path):
    fx = FX[case]
    lab, res, split = write_case(fx, str(tmp_path))
    texts = kitti_eval.evaluate(lab, res, split, [int(c) for c in fx["classes"]], gpu=0)
    assert texts == [str(t) for t in fx["texts"]]


def test_two_runs_are_identical(tmp_path):
    fx = FX["mixed"]
    a = run_case(fx, tmp_path / "a")
    b = run_case(fx, tmp_path / "b")
    for m in kitti_eval.METRICS:
        for k in ("precision", "thresholds", "orientation"):
            assert np.array_equal(a[m][k], b[m][k], equal_nan=True), (m, k)
    assert all(np.array_equal(x, y) for x, y in zip(a["overlaps"], b["overlaps"]))
