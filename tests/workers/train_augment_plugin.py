"""Worker of tests/test_train_augment_gpu.py::test_plugin_matches_the_reference_training_input (own process, GPU box).

Writes a two-frame KITTI tree under the directory given as argv[1] (PNG frames of two KITTI sizes, calib and label text, disparity PNGs,
an `imdb.pkl` of the reference's own KittiData) and runs, from the same numpy seed, the reference's KittiStereoDataset + collate_fn +
train_stereo_detection (Stereo3D_example's list) and KittiMonoDataset + collate_fn + train_mono_detection (Yolo3D_example's list), first
as shipped and then after `plugin.install_train_augmentation_into_reference()`.  A recording stub module stands in for the detector.
Prints one JSON line: per arm, the largest image difference, whether every other input the module got (annotations, P2 / P3,
disparity) is equal, and whether the numpy RNG ends at the same position."""
import json
import os
import pickle
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402
import refload  # noqa: E402
import train_augment_cases as cases  # noqa: E402

SIZES = [(375, 1242), (370, 1224)]


def write_tree(tmp, sizes=SIZES):
    from visualDet3D.data.kitti.kittidata import KittiCalib, KittiData, KittiObj
    raw, pre = os.path.join(tmp, "kitti", "training"), os.path.join(tmp, "pre")
    for d in ("calib", "image_2", "image_3", "label_2"):
        os.makedirs(os.path.join(raw, d), exist_ok=True)
    os.makedirs(os.path.join(pre, "training", "disp"), exist_ok=True)
    imdb = []
    for i, (H, W) in enumerate(sizes):
        idx = "%06d" % i
        cv2.imwrite(os.path.join(raw, "image_2", idx + ".png"), cases.frame(10 + i, H, W))
        cv2.imwrite(os.path.join(raw, "image_3", idx + ".png"), cases.frame(20 + i, H, W))
        fmt = lambda a: " ".join("%.12e" % v for v in np.asarray(a).reshape(-1))
        with open(os.path.join(raw, "calib", idx + ".txt"), "w") as f:
            f.write(f"P0: {fmt(cases.P2)}\nP1: {fmt(cases.P2)}\nP2: {fmt(cases.P2)}\nP3: {fmt(cases.P3)}\n"
                    f"R0_rect: {fmt(np.eye(3))}\nTr_velo_to_cam: {fmt(np.eye(3, 4))}\nTr_imu_to_velo: {fmt(np.eye(3, 4))}\n")
        objs = cases.labels(30 + i, H, W, KittiObj)
        with open(os.path.join(raw, "label_2", idx + ".txt"), "w") as f:
            for o in objs:
                f.write(f"Car 0.00 0 {o.alpha:.6f} {o.bbox_l:.2f} {o.bbox_t:.2f} {o.bbox_r:.2f} {o.bbox_b:.2f} {o.h:.2f} {o.w:.2f} "
                        f"{o.l:.2f} {o.x:.2f} {o.y:.2f} {o.z:.2f} {o.ry:.2f}\n")
        rng = np.random.RandomState(40 + i)
        for cam in ("P2", "P3"):
            cv2.imwrite(os.path.join(pre, "training", "disp", f"{cam}{idx}.png"), rng.randint(0, 96 * 16, (72, 320)).astype(np.uint16))
        kd = KittiData(raw, idx, {"calib": True, "image": False, "label": True, "velodyne": False})
        kd.calib, _, kd.label, _ = kd.read_data()
        kd.label = kd.label.data
        imdb.append(kd)
    with open(os.path.join(pre, "training", "imdb.pkl"), "wb") as f:
        pickle.dump(imdb, f)
    return pre


class Recorder(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.p = torch.nn.Parameter(torch.zeros(1, device="cuda"))
        self.seen = None

    def forward(self, inputs):
        self.seen = [x.detach().cpu() if torch.is_tensor(x) else x for x in inputs]
        s = self.p.sum()
        return s + 1.0, s, {}


def run(cfg, ds_cls, fn_name, seed):
    from visualDet3D.networks.utils import registry as ref
    ds = ds_cls(cfg, "training")
    np.random.seed(seed)
    data = ds_cls.collate_fn([ds[i] for i in range(len(SIZES))])
    module = Recorder()
    ref.PIPELINE_DICT[fn_name](data, module, torch.optim.SGD(module.parameters(), lr=0.1), cfg=cfg)
    torch.cuda.synchronize()
    return module.seen, np.random.rand(), type(ds.transform).__name__


def main():
    from visualdet3d_b200 import plugin
    from visualdet3d_b200.ops import dcn as our_dcn, iou3d as our_iou
    refload.load_reference(device="cuda", dcn_ext=our_dcn, iou3d_ext=our_iou)
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from make_golden_train_augment import edict
    from visualDet3D.data.kitti.dataset.mono_dataset import KittiMonoDataset
    from visualDet3D.data.kitti.dataset.stereo_dataset import KittiStereoDataset
    pre = write_tree(sys.argv[1])
    arms = {"stereo": (KittiStereoDataset, "train_stereo_detection", "stereo3d", (0, 1)),
            "mono": (KittiMonoDataset, "train_mono_detection", "yolo3d", (0, ))}
    res = {}
    for seed in (0, 3):                                   # two seeds: mirrored and unmirrored samples in each arm
        for arm, (cls, fn, name, img_slots) in arms.items():
            cfg = edict({"path": {"preprocessed_path": pre}, "obj_types": ["Car"],
                         "data": {"augmentation": {}, "train_augmentation": cases.LISTS[name][0], "use_right_image": False},
                         "optimizer": {"clipped_gradient_norm": 1.0}})
            res[f"{arm}_{seed}"] = [run(cfg, cls, fn, seed)]
    plugin.install_train_augmentation_into_reference()
    out = {}
    for seed in (0, 3):
        for arm, (cls, fn, name, img_slots) in arms.items():
            cfg = edict({"path": {"preprocessed_path": pre}, "obj_types": ["Car"],
                         "data": {"augmentation": {}, "train_augmentation": cases.LISTS[name][0], "use_right_image": False},
                         "optimizer": {"clipped_gradient_norm": 1.0}})
            (ref_seen, ref_next, ref_tf), = res[f"{arm}_{seed}"]
            seen, nxt, tf = run(cfg, cls, fn, seed)
            img = max(float((seen[k].float() - ref_seen[k].float()).abs().max()) for k in img_slots)
            shapes = all(seen[k].shape == ref_seen[k].shape for k in range(len(seen)))
            others = all(torch.equal(seen[k].float(), ref_seen[k].float()) for k in range(len(seen)) if k not in img_slots)
            on_gpu = all(seen[k].dtype == torch.float32 for k in img_slots)
            out[f"{arm}_{seed}"] = {"image_max_diff": img, "shapes_equal": shapes, "others_equal": others, "rng_equal": nxt == ref_next,
                                    "float_images": on_gpu, "n_inputs": len(seen),
                                    "transforms": [ref_tf, tf]}
    print("SEAM_JSON " + json.dumps(out))


if __name__ == "__main__":
    main()
