"""-m gpu: the native KITTI evaluator on the hand-written edge scenes (overlaps exactly at a minimum overlap, tied overlaps and scores, the
height / occlusion / truncation limits, DontCare regions, empty images, 70 detections in one image), against the unmodified reference
evaluator's stored outputs: what tests/test_kitti_eval_gpu.py asserts on its random scenes."""
import numpy as np
import pytest

from test_kitti_eval_cpu import write_case
from test_kitti_eval_edges_cpu import CASES, FX
from test_kitti_eval_gpu import BEV_TOL, run_case
from visualdet3d_b200 import kitti_eval

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", CASES)
def test_edge_scenes_match_reference(case, tmp_path):
    fx = FX[case]
    assert float(fx["margin"]) > 2 * BEV_TOL
    out = run_case(fx, tmp_path)
    got = np.concatenate([o.reshape(3, -1) for o in out["overlaps"]], 1)
    assert np.array_equal(got[0], fx["overlaps"][0])                       # bbox: bit-identical, ties and at-threshold values included
    assert np.abs(got[1:] - fx["overlaps"][1:]).max() < BEV_TOL
    for m in kitti_eval.METRICS:
        assert np.array_equal(out[m]["precision"], fx[f"{m}_precision"]), m
        assert np.array_equal(out[m]["thresholds"], fx[f"{m}_thresholds"]), m
    o, r = out["bbox"]["orientation"], fx["bbox_orientation"]
    assert np.allclose(o, r, rtol=1e-12, atol=0) and np.array_equal(o == 0, r == 0)


@pytest.mark.parametrize("case", CASES)
def test_edge_scenes_return_reference_text(case, tmp_path):
    fx = FX[case]
    lab, res, split = write_case(fx, str(tmp_path))
    assert kitti_eval.evaluate(lab, res, split, [int(c) for c in fx["classes"]], gpu=0) == [str(t) for t in fx["texts"]]
