"""Host side of the native KITTI evaluator (visualdet3d_b200/kitti_eval.py): label / result parsing and the printed AP text, against the
unmodified reference evaluator's outputs stored by tests/golden/make_golden_kitti_eval.py, and the seam that rebinds the reference's
`evaluate` to it."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from conftest import ROOT, load_fixture
import refload
from visualdet3d_b200 import kitti_eval

FX = load_fixture("kitti_eval")
CASES = sorted(k for k in FX if k != "riou")


def write_case(fx, root):
    """The case's label / result / split files under root; returns (label_path, result_path, split_file)."""
    lab, res = os.path.join(root, "label_2"), os.path.join(root, "data")
    os.makedirs(lab)
    os.makedirs(res)
    for i, l, r in zip(fx["ids"], fx["label_text"], fx["result_text"]):
        with open(os.path.join(lab, f"{int(i):06d}.txt"), "w") as f:
            f.write(str(l))
        with open(os.path.join(res, f"{int(i):06d}.txt"), "w") as f:
            f.write(str(r))
    split = os.path.join(root, "val.txt")
    with open(split, "w") as f:
        f.write("".join(f"{int(i):06d}\n" for i in fx["ids"]))
    return lab, res, split


@pytest.mark.parametrize("case", CASES)
def test_get_label_annos_matches_reference(case, tmp_path):
    fx = FX[case]
    lab, res, _ = write_case(fx, str(tmp_path))
    gt = kitti_eval.get_label_annos(lab, [int(i) for i in fx["ids"]])
    dt = kitti_eval.get_label_annos(res)            # the glob + sort path
    for who, annos in (("gt", gt), ("dt", dt)):
        assert [len(a["name"]) for a in annos] == fx["ng" if who == "gt" else "nd"].tolist()
        assert [n for a in annos for n in a["name"]] == fx[f"{who}_name"].tolist()
        for k in ("truncated", "occluded", "alpha", "bbox", "dimensions", "location", "rotation_y", "score"):
            got = np.concatenate([a[k] for a in annos], 0)
            assert got.dtype == fx[f"{who}_{k}"].dtype and np.array_equal(got, fx[f"{who}_{k}"]), (who, k)


@pytest.mark.parametrize("case", CASES)
def test_format_reproduces_reference_text(case, tmp_path):
    fx = FX[case]
    _, res, _ = write_case(fx, str(tmp_path))
    compute_aos = kitti_eval._compute_aos(kitti_eval.get_label_annos(res))
    assert compute_aos == (case != "bbox2d")
    for j, c in enumerate(fx["classes"]):
        metrics = {m: {"precision": fx[f"{m}_precision"][j:j + 1]} for m in kitti_eval.METRICS}
        metrics["bbox"]["orientation"] = fx["bbox_orientation"][j:j + 1]
        assert kitti_eval.format_official_result(metrics, int(c), compute_aos) == str(fx["texts"][j])


@pytest.mark.skipif(not refload.available(), reason="no reference package (neither /root/reference nor oracle/_ref/visualDet3D)")
def test_install_evaluator_into_reference():
    # own process: importing the reference patches torch globally
    code = textwrap.dedent(f"""
        import sys
        sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, "oracle")!r}]
        import refload
        refload.load_reference()
        from visualDet3D.networks.pipelines import evaluators
        import visualDet3D.evaluator.kitti.evaluate as ke
        from visualdet3d_b200 import plugin, kitti_eval
        before = (evaluators.evaluate, ke.evaluate)
        plugin.install_evaluator_into_reference()
        assert before[0] is before[1] and before[0] is not kitti_eval.evaluate
        assert evaluators.evaluate is kitti_eval.evaluate and ke.evaluate is kitti_eval.evaluate
        print("REBOUND")
    """)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "REBOUND" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
