"""Golden outputs for Stereo3D's disparity ground truth (tests/disparity_gt_cases.py):
  bm/<case>      cv2.StereoBM_create(192, 25).compute(left, right), int16 (cv2's version in `cv2_version`)
  bmr/<case>     skimage.measure.block_reduce(max(bm, 0) as uint16, (4, 4), np.max)
  velo/<case>    the reference's generate_dispariy_from_velo (R/data/kitti/utils.py:85-120), uint16
  velor/<case>   its 4x4 block max
  tree_bm/<P2|P3><n>, tree_velo/<P2|P3><n>
                 the decoded PNGs the UNMODIFIED reference scripts/disparity_compute.py (compute_dispairity_for_split) writes for the
                 constructed KITTI tree (disparity_gt_cases.write_tree), StereoBM and LiDAR modes.
Two import shims, no reference source edited: `fire` is only used under the script's __main__, and skimage.measure.block_reduce (the stub
package of oracle/refload.py is empty) is given a max-with-zero-pad stand-in, which is what block_reduce(.., np.max) computes on
non-negative arrays.  `coloredlogs` (imported by scripts/_path_init.py) is stubbed likewise.
The zip members carry a fixed timestamp, so a second run writes the same bytes.   python tests/golden/make_golden_disparity_gt.py"""
import importlib.util
import io
import os
import sys
import tempfile
import types
import zipfile

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (os.path.dirname(HERE), ROOT, os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)
import disparity_gt_cases as dc  # noqa: E402
import refload  # noqa: E402
import stereo_bm as sb  # noqa: E402

OUT = os.path.join(HERE, "disparity_gt.npz")


def block_reduce(image, block_size, func=np.max):
    assert func is np.max and tuple(block_size) == (4, 4)
    return sb.block_max(image)


def reference_script():
    refload.load_reference()
    sys.modules["fire"] = types.SimpleNamespace(Fire=None)
    sys.modules.setdefault("coloredlogs", types.ModuleType("coloredlogs"))
    sys.modules["skimage.measure"].block_reduce = block_reduce
    sys.modules["skimage"].measure = sys.modules["skimage.measure"]
    scripts = os.path.join(refload.ref_root(), "scripts")
    sys.path.insert(0, scripts)
    spec = importlib.util.spec_from_file_location("ref_disparity_compute", os.path.join(scripts, "disparity_compute.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def run_tree(mod, use_point_cloud):
    from visualDet3D.utils.utils import cfg_from_file
    with tempfile.TemporaryDirectory() as tmp:
        cfg = cfg_from_file(dc.write_tree(tmp))
        names, _ = mod.process_train_val_file(cfg)
        output_dict = {"calib": True, "image": True, "image_3": True, "label": False, "velodyne": use_point_cloud}
        mod.compute_dispairity_for_split(cfg, names, cfg.path.data_path, output_dict, 'training', 100, use_point_cloud)
        disp = os.path.join(cfg.path.preprocessed_path, "training", "disp")
        return {f[:-4]: cv2.imread(os.path.join(disp, f), -1) for f in sorted(os.listdir(disp))}


def main():
    mod = reference_script()
    from visualDet3D.data.kitti.utils import generate_dispariy_from_velo
    out = {"cv2_version": np.array(cv2.__version__)}
    matcher = cv2.StereoBM_create(192, 25)
    for c in dc.bm_cases():
        d = matcher.compute(c["left"], c["right"])
        out["bm/" + c["id"]] = d
        out["bmr/" + c["id"]] = block_reduce(np.maximum(d, 0).astype(np.uint16), (4, 4), np.max)
    for c in dc.velo_cases():
        v = generate_dispariy_from_velo(c["points"][:, 0:3], c["H"], c["W"], c["Tr_velo_to_cam"], c["R0_rect"], c["P2"],
                                        baseline=c["baseline"])
        out["velo/" + c["id"]] = v
        out["velor/" + c["id"]] = block_reduce(v, (4, 4), np.max)
    for mode, pc in (("tree_bm", False), ("tree_velo", True)):
        for k, a in run_tree(mod, pc).items():
            out[f"{mode}/{k}"] = a
    with zipfile.ZipFile(OUT, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(out):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asarray(out[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(2020, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())
    print("wrote", OUT, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
