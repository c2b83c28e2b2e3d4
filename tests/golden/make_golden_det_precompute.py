"""Golden outputs for the det_precompute CLI and the anchor-prior accumulation (tests/det_precompute_cases.py):
  case/<id>/{examine,sums,squared,usable}   each constructed kernel case's accumulator state, from the reference's own calc_iou and
                                            torch.max and the script's loop (imdb_precompute_3d.py:110-135) on the CPU
  <config>/<split>/anchor_{mean,std}_<type>  the arrays the UNMODIFIED reference scripts/imdb_precompute_3d.py writes for the constructed
                                            tree (det_precompute_cases.write_tree) under each config of det_precompute_cases.CONFIGS
  <config>/<split>/pkl/...                   its imdb.pkl flattened: the KittiData paths (tree root replaced by <ROOT>), output_dict,
                                            every label field and the calibration matrices
  test/test/pkl/...                          imdb_precompute_test.py's pickle, likewise
Environment shims only, no reference source edited: `fire` and `coloredlogs` (imported under the scripts' __main__ and by _path_init.py)
are stubbed, and torch.ones maps device="cuda" to the CPU (Anchors.forward, anchors.py:113, allocates its mask there).
The zip members carry a fixed timestamp, so a second run writes the same bytes.   python tests/golden/make_golden_det_precompute.py"""
import importlib.util
import io
import os
import pickle
import sys
import tempfile
import types
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (os.path.dirname(HERE), ROOT, os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)
import det_precompute_cases as dc  # noqa: E402
import refload  # noqa: E402

OUT = os.path.join(HERE, "det_precompute.npz")
LABEL_FIELDS = ("truncated", "occluded", "alpha", "bbox_l", "bbox_t", "bbox_r", "bbox_b", "h", "w", "l", "x", "y", "z", "ry")
CALIB_FIELDS = ("P2", "P3", "R0_rect", "Tr_velo_to_cam")


def reference_scripts(scripts_dir=None, cpu=True):
    """The two scripts as modules.  cpu: load the reference in CPU mode and map torch.ones(device="cuda") to the CPU; otherwise the
    caller has loaded it on the GPU already."""
    if cpu:
        refload.load_reference()
    sys.modules["fire"] = types.SimpleNamespace(Fire=None)
    sys.modules.setdefault("coloredlogs", types.ModuleType("coloredlogs"))
    import torch
    if cpu and not getattr(torch.ones, "_cpu_shim", False):
        ones = torch.ones

        def cpu_ones(*a, device=None, **k):
            return ones(*a, device=None if device == "cuda" else device, **k)
        cpu_ones._cpu_shim = True
        torch.ones = cpu_ones
    scripts = scripts_dir or os.path.join(refload.ref_root(), "scripts")
    sys.path.insert(0, scripts)
    mods = []
    for name in ("imdb_precompute_3d", "imdb_precompute_test"):
        spec = importlib.util.spec_from_file_location("ref_" + name, os.path.join(scripts, name + ".py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        mods.append(mod)
    return mods


def flatten_pickle(path, root, prefix, out):
    """imdb.pkl as arrays: per-frame paths / output_dict as strings, label fields as float64 columns with a per-frame count."""
    with open(path, "rb") as f:
        frames = pickle.load(f)
    attrs = sorted(vars(frames[0]).keys()) if frames else []
    out[prefix + "attrs"] = np.array(attrs)
    for a in ("calib_path", "image2_path", "image3_path", "label2_path", "velodyne_path"):
        out[prefix + a] = np.array([getattr(fr, a).replace(root, "<ROOT>") for fr in frames])
    out[prefix + "output_dict"] = np.array([repr(sorted(fr.output_dict.items())) for fr in frames])
    labels = [getattr(fr, "label", None) or [] for fr in frames]
    out[prefix + "n_labels"] = np.array([len(lb) for lb in labels], dtype=np.int64)
    out[prefix + "label_type"] = np.array([o.type for lb in labels for o in lb] or [""])
    for k in LABEL_FIELDS:
        out[prefix + "label_" + k] = np.array([getattr(o, k) for lb in labels for o in lb], dtype=np.float64)
    for k in CALIB_FIELDS:
        out[prefix + "calib_" + k] = np.stack([np.asarray(getattr(fr.calib, k), dtype=np.float64) for fr in frames])
    out[prefix + "has_label"] = np.array([hasattr(fr, "label") for fr in frames])


def reference_state(case):
    """The script's lines 110-135 on one constructed batch: calc_iou, torch.max, the python loop over positives."""
    import torch
    from visualDet3D.networks.utils.utils import calc_iou
    T, nb = case["T"], case["n_bins"]
    examine = np.zeros((T, nb), np.int64)
    sums = np.zeros((T, nb, 3))
    squared = np.zeros((T, nb, 3))
    usable = np.zeros(T, np.int64)
    anchors = torch.tensor(case["anchors"])
    off = case["offsets"]
    for s in range(case["B"] * T):
        t = s % T
        rows = case["boxes"][off[s]:off[s + 1]]
        if len(rows) < 1:
            continue
        bbox2d = torch.tensor(rows.tolist(), dtype=torch.float64 if case["f64"] else torch.float32)
        bbox3d = torch.tensor(case["gt3"][off[s]:off[s + 1]])
        IoUs = calc_iou(anchors, bbox2d)
        IoU_max, _ = torch.max(IoUs, dim=0)
        IoU_max_anchor, IoU_argmax_anchor = torch.max(IoUs, dim=1)
        usable[t] += torch.sum(IoU_max > case["thr"]).item()
        mask = IoU_max_anchor > case["thr"]
        g = bbox3d[IoU_argmax_anchor[mask]].numpy()
        bins = case["bins"][mask.numpy()]
        for k in range(len(bins)):
            examine[t, bins[k]] += 1
            sums[t, bins[k]] += g[k]
            squared[t, bins[k]] += g[k] ** 2
    return dict(examine=examine, sums=sums, squared=squared, usable=usable)


def run_reference(mod3d, modtest, tmp, raw, split, out):
    from visualDet3D.utils.utils import cfg_from_file
    for name in dc.CONFIGS:
        cfg = cfg_from_file(dc.write_config(name, tmp, raw, split))
        tr, va = mod3d.process_train_val_file(cfg)
        mod3d.read_one_split(cfg, tr, raw, {"calib": True, "image": True, "label": True, "velodyne": False}, 'training', 100)
        mod3d.read_one_split(cfg, va, raw, {"calib": True, "image": False, "label": True, "velodyne": False}, 'validation', 100)
        for sp in ("training", "validation"):
            d = os.path.join(cfg.path.preprocessed_path, sp)
            for f in sorted(os.listdir(d)):
                if f.endswith(".npy"):
                    out[f"{name}/{sp}/{f[:-4]}"] = np.load(os.path.join(d, f))
            flatten_pickle(os.path.join(d, "imdb.pkl"), tmp, f"{name}/{sp}/pkl/", out)
    cfg = cfg_from_file(dc.write_config("stereo3d", tmp, raw, split))
    root = cfg.path.test_path
    names = ["%06d" % i for i in range(len(os.listdir(os.path.join(root, 'calib'))))]
    modtest.read_one_split(cfg, names, root, {"calib": True, "image": False, "label": False, "velodyne": False}, 'test', 100)
    flatten_pickle(os.path.join(cfg.path.preprocessed_path, "test", "imdb.pkl"), tmp, "test/test/pkl/", out)


def main():
    mod3d, modtest = reference_scripts()
    out = {}
    for c in dc.kernel_cases():
        for k, v in reference_state(c).items():
            out[f"case/{c['id']}/{k}"] = v
    with tempfile.TemporaryDirectory() as tmp:
        raw, split = dc.write_tree(tmp)
        run_reference(mod3d, modtest, tmp, raw, split, out)
    with zipfile.ZipFile(OUT, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(out):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asarray(out[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(2020, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())
    print("wrote", OUT, len(out), "arrays")


if __name__ == "__main__":
    main()
