"""The hand-written edge scenes of tests/golden/make_golden_kitti_eval_edges.py still contain what they claim (overlaps exactly at the
minimum overlap, ties, a 70-detection image, more than 41 true-positive scores), and the host parser reproduces the stored annos."""
import numpy as np
import pytest

import rotated_cases as rc
from conftest import load_fixture
from test_kitti_eval_cpu import write_case
from visualdet3d_b200 import kitti_eval

FX = load_fixture("kitti_eval_edges")
CASES = ("edges", "single")


def image_overlaps(fx, scene):
    """[3][dt][gt] of one named scene of the `edges` case."""
    i = FX["edges"]["scenes"].tolist().index(scene)
    o = np.concatenate([[0], np.cumsum(fx["ng"] * fx["nd"])])
    return fx["overlaps"][:, o[i]:o[i + 1]].reshape(3, fx["nd"][i], fx["ng"][i])


def test_fixture_holds_its_edges():
    fx = FX["edges"]
    assert len(fx["ids"]) < 50 and len(FX["single"]["ids"]) == 1
    car, ped = image_overlaps(fx, "thr_car")[0], image_overlaps(fx, "thr_ped")[0]
    assert car[0, 0] == 0.7 and car[1, 1] == 15 / 19 and car[2, 2] == 13 / 21          # at the Car minimum overlap, and either side
    assert ped[0, 0] == 0.5 and ped[2, 1] == 7 / 11 and ped[4, 2] == 5 / 13
    ties = image_overlaps(fx, "ties")[0]
    assert ties[0, 0] == ties[1, 0] > 0.7 and ties[2, 1] == ties[3, 1] > 0.7 and ties[4, 2] == ties[4, 3] > 0.7
    assert 70 in fx["nd"].tolist() and fx["ng"][fx["nd"].tolist().index(70)] == 45    # three 32-bit flag words, more than 41 matches
    assert 0 in (fx["ng"] + fx["nd"]).tolist() and ((fx["ng"] == 0) & (fx["nd"] > 0)).any() and ((fx["nd"] == 0) & (fx["ng"] > 0)).any()
    heights = fx["gt_bbox"][:, 3] - fx["gt_bbox"][:, 1]
    assert {25.0, 26.0, 40.0, 41.0} <= set(heights.tolist()) and {24.0, 25.0, 39.0, 40.0} <= set((fx["dt_bbox"][:, 3] - fx["dt_bbox"][:, 1]).tolist())
    assert {0.15, 0.16, 0.3, 0.31, 0.5, 0.51} <= set(fx["gt_truncated"].tolist()) and {0, 1, 2, 3} <= set(fx["gt_occluded"].tolist())
    assert "Cyclist" in fx["dt_name"] and "Cyclist" not in fx["gt_name"] and "DontCare" in fx["gt_name"] and "Van" in fx["gt_name"]
    bev = image_overlaps(fx, "bev")[1]
    turned = rc.octagon_area(4, 2, 0.5)                                     # closed forms of tests/rotated_cases.py at KITTI range
    assert abs(bev[0, 0] - 1.0) < 1e-6 and abs(bev[1, 1] - turned / (16 - turned)) < 1e-4 and abs(bev[2, 2] - 2 / 30) < 1e-4
    assert (fx["bbox_thresholds"] > 0).sum(-1).max() >= 38                                # far more true positives than the 41 recall points sample
    for case in CASES:
        assert float(FX[case]["margin"]) > 1e-4


@pytest.mark.parametrize("case", CASES)
def test_parser_reproduces_stored_annos(case, tmp_path):
    fx = FX[case]
    lab, res, _ = write_case(fx, str(tmp_path))
    for who, annos in (("gt", kitti_eval.get_label_annos(lab, [int(i) for i in fx["ids"]])), ("dt", kitti_eval.get_label_annos(res))):
        assert [len(a["name"]) for a in annos] == fx["ng" if who == "gt" else "nd"].tolist()
        assert [n for a in annos for n in a["name"]] == fx[f"{who}_name"].tolist()
        for k in ("truncated", "occluded", "alpha", "bbox", "dimensions", "location", "rotation_y", "score"):
            assert np.array_equal(np.concatenate([a[k] for a in annos], 0), fx[f"{who}_{k}"]), (who, k)
