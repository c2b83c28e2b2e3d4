"""Stereo3D's disparity precompute on the GPU: the reference's scripts/disparity_compute.py (run by launchers/disparity_precompute.sh)
with the StereoBM or LiDAR maps computed by csrc/disparity_gt.cu.

    python -m visualdet3d_b200.disparity_precompute --config=config/Stereo3D_example.py --use_point_cloud=False

writes `P2%06d.png` and `P3%06d.png` (numbered in the train split's order) under `cfg.path.preprocessed_path/training/disp`, with the
same decoded arrays as the reference script.  The host work stays the reference's own: `cfg_from_file`, `KittiData` and
`build_augmentator(cfg.data.test_augmentation)`, imported from the reference package (an ImportError means it is not on sys.path).  The
test augmentation's float32 output must stay the reference's to the bit: the script's denorm truncates, so a one-ulp difference on a
flat region can change a grey level.  A small thread pool decodes and augments the next batch (cv2 and PIL release the GIL) while the
device works on the current one, and writes the PNGs.

Two of the reference's quirks are kept on purpose:
  - the P3 file holds the LEFT map, as the reference writes it (disparity_compute.py:111-113).  The reference's right-image map is
    computed and then discarded, so it is not computed here; nothing observable changes.  `disparity_gt.stereo_bm` on mirrored frames
    gives a right map to anyone who wants one.
  - the numbering is the enumeration index in the split file, not the KITTI index."""
from __future__ import annotations

import argparse
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor
from copy import deepcopy
from typing import Dict, List

import cv2
import numpy as np
import torch

from . import disparity_gt

BATCH = 8
WORKERS = 4


def process_train_val_file(cfg):
    """The reference script's split reader: (train names, val names), stripped lines."""
    names = []
    for path in (cfg.data.train_split_file, cfg.data.val_split_file):
        with open(path) as f:
            names.append([line.strip() for line in f.readlines()])
    return names[0], names[1]


def compute_dispairity_for_split(cfg, index_names: List[str], data_root_dir: str, output_dict: Dict, data_split: str = 'training',
                                 time_display_inter: int = 100, use_point_cloud: bool = True):
    """The reference's function of the same name and signature, with the maps computed on the current CUDA device."""
    from visualDet3D.data.pipeline import build_augmentator         # ImportError if the reference is not on sys.path
    from visualDet3D.data.kitti.kittidata import KittiData

    save_dir = os.path.join(cfg.path.preprocessed_path, data_split)
    if not os.path.isdir(save_dir):
        os.makedirs(save_dir)
    disp_dir = os.path.join(save_dir, 'disp')
    if not os.path.isdir(disp_dir):
        os.mkdir(disp_dir)
    preprocess = build_augmentator(cfg.data.test_augmentation)
    mean, std = cfg.data.augmentation.rgb_mean, cfg.data.augmentation.rgb_std

    def load(i):
        calib, image, right_image, label, velo = KittiData(data_root_dir, index_names[i], output_dict).read_data()
        baseline = (calib.P2[0, 3] - calib.P3[0, 3]) / calib.P2[0, 0]
        image, image_3, P2, P3 = preprocess(image.copy(), right_image.copy(), p2=deepcopy(calib.P2), p3=deepcopy(calib.P3))
        return dict(image=np.ascontiguousarray(image, np.float32), image_3=np.ascontiguousarray(image_3, np.float32), P2=P2, calib=calib,
                    velo=velo, baseline=baseline)

    def write(i, disparity):
        for cam in ("P2", "P3"):                                     # the reference writes the left map into both files
            if not cv2.imwrite(os.path.join(disp_dir, "%s%06d.png" % (cam, i)), disparity):
                raise OSError(f"cv2.imwrite failed under {disp_dir}")

    def compute(frames):
        """The maps of one batch, as host uint16 arrays."""
        if use_point_cloud:
            outs = []
            for f in frames:
                pts = torch.from_numpy(np.ascontiguousarray(f["velo"][:, 0:3])).cuda()
                H, W = f["image"].shape[:2]
                outs.append(disparity_gt.velo_targets(pts, f["calib"].R0_rect, f["calib"].Tr_velo_to_cam, f["P2"], f["baseline"], H, W))
            return [o.cpu().numpy() for o in outs]
        outs = []
        start = 0
        while start < len(frames):                                   # one launch per run of equally sized frames
            shape = frames[start]["image"].shape
            end = start
            while end < len(frames) and frames[end]["image"].shape == shape:
                end += 1
            left = torch.from_numpy(np.stack([f["image"] for f in frames[start:end]])).pin_memory().cuda(non_blocking=True)
            right = torch.from_numpy(np.stack([f["image_3"] for f in frames[start:end]])).pin_memory().cuda(non_blocking=True)
            outs.extend(disparity_gt.bm_targets(left, right, mean, std).cpu().numpy())
            start = end
        return outs

    N = len(index_names)
    print("start reading {} data".format(data_split))
    t0 = time.time()
    with ThreadPoolExecutor(WORKERS) as pool:
        batches = [list(range(s, min(s + BATCH, N))) for s in range(0, N, BATCH)]
        pending = [pool.submit(load, i) for i in batches[0]] if batches else []
        writes = []
        for b, idx in enumerate(batches):
            frames = [p.result() for p in pending]
            pending = [pool.submit(load, i) for i in batches[b + 1]] if b + 1 < len(batches) else []
            for i, disparity in zip(idx, compute(frames)):
                writes.append(pool.submit(write, i, disparity))
            done = idx[-1] + 1
            if done // time_display_inter != (done - len(idx)) // time_display_inter or done == N:
                print("{}/{} frames, {:.1f} frames/s".format(done, N, done / max(time.time() - t0, 1e-9)))
        for w in writes:
            w.result()
    print("{} split finished precomputing disparity".format(data_split))


def _bool(text: str) -> bool:
    t = text.strip().lower()
    if t in ("true", "1", "yes"):
        return True
    if t in ("false", "0", "no"):
        return False
    raise argparse.ArgumentTypeError(f"expected True or False, got {text!r}")


def parse_args(argv=None):
    ap = argparse.ArgumentParser(prog="python -m visualdet3d_b200.disparity_precompute",
                                 description="Stereo3D's disparity ground truth (the reference's disparity precompute) on the GPU.")
    ap.add_argument("--config", default="config/config.py", help="the reference's config file (.py)")
    ap.add_argument("--use_point_cloud", type=_bool, nargs="?", const=True, default=False,
                    help="True: project the velodyne cloud; False (default): StereoBM on the stereo pair")
    args = ap.parse_args(argv)
    if not args.config.endswith(".py"):
        ap.error(f"--config must name a .py config file, got {args.config!r}")
    return args


def main(config: str = "config/config.py", use_point_cloud: bool = False):
    """The reference script's main: the training split's disparity maps."""
    from visualDet3D.utils.utils import cfg_from_file                # ImportError if the reference is not on sys.path
    cfg = cfg_from_file(config)
    torch.cuda.set_device(cfg.trainer.gpu)
    data_root_dir = cfg.path.data_path
    output_dict = {"calib": True, "image": True, "image_3": True, "label": False, "velodyne": use_point_cloud}
    train_names, _ = process_train_val_file(cfg)
    compute_dispairity_for_split(cfg, train_names, data_root_dir, output_dict, 'training', 100, use_point_cloud)
    print("Preprocessing finished")


if __name__ == "__main__":
    a = parse_args(sys.argv[1:])
    main(a.config, a.use_point_cloud)
