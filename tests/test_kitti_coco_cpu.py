"""Host side of the COCO-style KITTI AP and of the evaluator's command line (visualdet3d_b200/kitti_eval.py): the min-overlap rows and
the printed text from the unmodified reference's stored curves (tests/golden/make_golden_kitti_coco.py), and the command line's
refusals, which exit non-zero with a message and no traceback; the library's checks on the number of min-overlap rows."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT, load_fixture
from test_kitti_eval_cpu import write_case
from visualdet3d_b200 import _lib, kitti_eval

FX = load_fixture("kitti_coco")
CASES = sorted(FX)


@pytest.mark.parametrize("case", CASES)
def test_coco_rows_match_reference(case):
    fx = FX[case]
    classes = [int(c) for c in fx["classes"]]
    assert np.array_equal(kitti_eval.coco_min_overlaps(kitti_eval._coco_overlap_ranges(classes)), fx["min_overlaps"])


@pytest.mark.parametrize("case", CASES)
def test_coco_format_reproduces_reference_text(case, tmp_path):
    fx = FX[case]
    _, res, _ = write_case(fx, str(tmp_path))
    compute_aos = kitti_eval._compute_aos(kitti_eval.get_label_annos(res))
    assert compute_aos == bool(fx["compute_aos"]) == (case != "bbox2d")
    if case == "occluded_cyclists":                        # Cyclist (class 2) has ground truth in moderate and hard only
        assert [bool(fx["bbox_precision"][2, d].any()) for d in range(3)] == [False, True, True]
    metrics = {m: {"precision": fx[f"{m}_precision"]} for m in kitti_eval.METRICS}
    metrics["bbox"]["orientation"] = fx["bbox_orientation"]
    classes = [int(c) for c in fx["classes"]]
    assert kitti_eval.format_coco_result(metrics, classes, compute_aos) == "".join(str(t) for t in fx["texts"])
    for j, c in enumerate(classes):
        one = {m: {k: v[j:j + 1] for k, v in d.items()} for m, d in metrics.items()}
        assert kitti_eval.format_coco_result(one, c, compute_aos) == str(fx["texts"][j])


def run_cli(*args):
    env = dict(os.environ, PYTHONPATH=ROOT)
    return subprocess.run([sys.executable, "-m", "visualdet3d_b200.kitti_eval", *args], capture_output=True, text=True, cwd=ROOT,
                          env=env, timeout=300)


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    return write_case(FX["mixed"], str(tmp_path_factory.mktemp("coco_cli")))


@pytest.mark.parametrize("extra, message", [
    (["--evaluator", "kitti_depth"], "depth evaluator"),
    (["--evaluator", "KITTI_Depth"], "depth evaluator"),
    (["--evaluator", "kitti_tracking"], "only kitti_obj"),
    (["--current_classes", "Truck"], "unknown class 'Truck'"),
    (["--current_classes", "0,9"], "unknown class '9'"),
    (["--current_classes", ""], "unknown class ''"),
    (["--gpu", "first"], "--gpu"),
    (["--label_split_file", "no_such_split.txt"], "--label_split_file"),
])
def test_cli_refuses_without_traceback(files, extra, message):
    lab, res, split = files
    r = run_cli("--label_path", lab, "--result_path", res, "--label_split_file", split, *extra)
    assert r.returncode != 0 and r.stdout == ""
    assert message in r.stderr and "Traceback" not in r.stderr, r.stderr


@pytest.mark.parametrize("missing", ["--label_path", "--result_path"])
def test_cli_requires_both_folders(files, missing):
    lab, res, split = files
    args = {"--label_path": lab, "--result_path": res, "--label_split_file": split}
    args.pop(missing)
    r = run_cli(*[x for kv in args.items() for x in kv])
    assert r.returncode != 0 and missing in r.stderr and "Traceback" not in r.stderr, r.stderr
    r = run_cli(*[x for kv in args.items() for x in kv], missing, os.path.join(lab, "no_such_folder"))
    assert r.returncode != 0 and "does not exist" in r.stderr and "Traceback" not in r.stderr, r.stderr


def test_row_count_is_validated():
    with pytest.raises(ValueError, match="no rows"):
        kitti_eval.DeviceEval([{"name": np.array([])}], [{"name": np.array([])}], [0], np.zeros((0, 3, 1)), False)
    lib = _lib.load()
    sizes = (4, 0, 20, 4)                                  # n_img, n_gt, n_dt, n_words: no scores to sort, so no CUDA query
    two = lib.vd3d_kitti_eval_workspace_bytes(*sizes, 3, 2)
    ten = lib.vd3d_kitti_eval_workspace_bytes(*sizes, 3, 10)
    assert 0 < two < ten
    for n_mo in (0, -1, 1 << 24):                          # 9 n_mo n_cls configurations must stay indexable
        assert lib.vd3d_kitti_eval_workspace_bytes(*sizes, 3, n_mo) == -1
        assert "kitti_eval_workspace_bytes" in lib.vd3d_last_error().decode()
    dummy = 1 << 12                                        # never dereferenced: the sizes are refused first
    rc = lib.vd3d_kitti_eval(dummy, dummy, dummy, 4, 0, 20, 0, 4, dummy, 3, dummy, 0, 0, dummy, dummy, dummy, dummy, dummy,
                             dummy, two, None)
    assert rc == -1 and "bad sizes" in lib.vd3d_last_error().decode()
