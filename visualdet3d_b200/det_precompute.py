"""The reference's det_precompute (launchers/det_precompute.sh: scripts/imdb_precompute_3d.py and imdb_precompute_test.py) with the
anchor priors computed on the GPU (anchor_prior.py, csrc/anchor_prior.cu).

    python -m visualdet3d_b200.det_precompute --config=config/Stereo3D_example.py --split=train
    python -m visualdet3d_b200.det_precompute --config=config/Stereo3D_example.py --split=test

`train` writes `imdb.pkl` under `cfg.path.preprocessed_path/{training,validation}` and, for configs with `anchor_prior` (the default),
`anchor_{mean,std}_{type}.npy` under `training`, equal to the reference script's files.  `test` writes `test/imdb.pkl` (no arithmetic,
host only).  `cfg_from_file`, `KittiData` and the label / calib parsing are the reference package's own, so the pickles hold its classes
(an ImportError means the reference is not on sys.path).

No frame is decoded when the test augmentation has a host geometry form (ConvertToFloat, CropTop, Resize, FilterObject, Normalize: every
anchor config's list): the script uses only the augmented image's shape, which follows from the PNG header, and the labels, which follow
from train_augment's host steps.  Any other list falls back to decoding the frame and running the reference's `build_augmentator`, as the
script does.  Label / calib parsing runs on a small thread pool; the batch of frames goes to the device whenever it reaches BATCH frames or
the post-augmentation shape changes, so the accumulation keeps the script's frame order."""
from __future__ import annotations

import argparse
import os
import pickle
import struct
import sys
import time
from concurrent.futures import ThreadPoolExecutor
from copy import deepcopy

import numpy as np
import torch

from . import train_augment
from .anchor_prior import AnchorPriorAccumulator

BATCH = 64
WORKERS = 4
_HOST_GEOMETRY = {"ConvertToFloat", "CropTop", "Resize", "FilterObject", "Normalize"}


def process_train_val_file(cfg):
    """The reference script's split reader: (train names, val names), stripped lines."""
    names = []
    for path in (cfg.data.train_split_file, cfg.data.val_split_file):
        with open(path) as f:
            names.append([line.strip() for line in f.readlines()])
    return names[0], names[1]


def png_shape(path: str):
    """(H, W) from a PNG's IHDR chunk, or None when the file is not a PNG."""
    with open(path, "rb") as f:
        head = f.read(24)
    if len(head) < 24 or head[:8] != b"\x89PNG\r\n\x1a\n" or head[12:16] != b"IHDR":
        return None
    w, h = struct.unpack(">II", head[16:24])
    return int(h), int(w)


class TestGeometry:
    """The test augmentation's effect on (shape, P2, labels).  With a host form (every step in _HOST_GEOMETRY and buildable there), the
    shape comes from the PNG header and train_augment's host steps update P2 / labels; otherwise the frame is decoded and the reference's
    own Compose runs on it."""

    def __init__(self, aug_list):
        self.host = all(c["type_name"] in _HOST_GEOMETRY for c in aug_list)
        if self.host:
            try:                                                        # steps with no host form: CropTop by output height,
                self.steps = [train_augment._build(c) for c in aug_list]   # Resize without preserve_aspect_ratio, ...
            except NotImplementedError:
                self.host = False
        if not self.host:
            from visualDet3D.data.pipeline import build_augmentator          # ImportError if the reference is not on sys.path
            self.compose = build_augmentator(aug_list)

    def __call__(self, image_path: str, p2: np.ndarray, labels: list):
        """(H, W) after the augmentation, the augmented P2 and labels (both copies)."""
        hw = png_shape(image_path) if self.host else None
        if hw is None:
            from visualDet3D.data.kitti.kittidata import read_image
            image = read_image(image_path)
            if self.host:
                hw = image.shape[:2]
            else:
                image, p2, labels = self.compose(image.copy(), p2=deepcopy(p2), labels=deepcopy(labels))
                return image.shape[:2], p2, labels
        st = train_augment._State()
        st.h, st.w = hw
        st.p2, st.p3, st.labels = deepcopy(p2), None, deepcopy(labels)
        for s in self.steps:
            s.apply(st)
        return (st.h, st.w), st.p2, st.labels


def read_one_split(cfg, index_names, data_root_dir, output_dict, data_split='training', time_display_inter=100, device="cuda"):
    """The reference's function of the same name and signature (imdb_precompute_3d.py:34-177), the anchor statistics on the current
    CUDA device (device=None: on the host, through the parity checker)."""
    from visualDet3D.data.kitti.kittidata import KittiData              # ImportError if the reference is not on sys.path
    save_dir = os.path.join(cfg.path.preprocessed_path, data_split)
    if not os.path.isdir(save_dir):
        os.makedirs(save_dir)
    if data_split == 'training':
        disp_dir = os.path.join(save_dir, 'disp')
        if not os.path.isdir(disp_dir):
            os.mkdir(disp_dir)

    N = len(index_names)
    frames = [None] * N
    print("start reading {} data".format(data_split))
    anchor_prior = getattr(cfg, 'anchor_prior', True) and data_split == 'training'
    max_occlusion = getattr(cfg.data, 'max_occlusion', 2)
    min_z = getattr(cfg.data, 'min_z', 3)
    geometry = TestGeometry(cfg.data.test_augmentation) if anchor_prior else None

    def load(i):
        data_frame = KittiData(data_root_dir, index_names[i], output_dict)
        data_frame.output_dict = dict(output_dict, image=False)        # the image is never decoded here ...
        calib, _, label, _ = data_frame.read_data()
        data_frame.output_dict = output_dict                            # ... but the pickle keeps the caller's dict
        if data_split == 'training':
            data_frame.label = [obj for obj in label.data if obj.type in cfg.obj_types and obj.occluded < max_occlusion and obj.z > min_z]
        else:
            data_frame.label = [obj for obj in label.data if obj.type in cfg.obj_types]
        data_frame.calib = calib
        aug = None
        if anchor_prior and len(data_frame.label) > 0:
            hw, _, labels = geometry(data_frame.image2_path, calib.P2, data_frame.label)
            aug = (tuple(hw), labels)
        return data_frame, aug

    acc = None
    if anchor_prior:
        head = cfg.detector.head
        acc = AnchorPriorAccumulator(head.anchors_cfg, None, cfg.obj_types, head.loss_cfg.fg_iou_threshold, device,
                                     getattr(cfg.detector, "name", "config"))
    batch, batch_hw = [], None
    t0 = time.time()
    with ThreadPoolExecutor(WORKERS) as pool:
        for i, (data_frame, aug) in enumerate(pool.map(load, range(N))):
            frames[i] = data_frame
            if anchor_prior:
                acc.count_objects(data_frame.label)
                if aug is not None:
                    if batch and (aug[0] != batch_hw or len(batch) == BATCH):
                        acc.add(batch, batch_hw)
                        batch = []
                    batch_hw = aug[0]
                    batch.append(aug[1])
            if (i + 1) % time_display_inter == 0 or i + 1 == N:
                print("{} {}/{} frames, {:.1f} frames/s".format(data_split, i + 1, N, (i + 1) / max(time.time() - t0, 1e-9)))
    if anchor_prior:
        if batch:
            acc.add(batch, batch_hw)
        for j, (avg, std) in enumerate(acc.finalize()):
            np.save(os.path.join(save_dir, 'anchor_mean_{}.npy'.format(cfg.obj_types[j])), avg)
            np.save(os.path.join(save_dir, 'anchor_std_{}.npy'.format(cfg.obj_types[j])), std)
        print("total_objs:{}, usable_objs:{}".format(acc.total_objects, acc.usable_objects()))
    with open(os.path.join(save_dir, 'imdb.pkl'), 'wb') as f:
        pickle.dump(frames, f)
    print("{} split finished precomputing".format(data_split))


def read_test_split(cfg, index_names, data_root_dir, output_dict, data_split='test', time_display_inter=100):
    """imdb_precompute_test.py's read_one_split: the calibration of every test frame, pickled."""
    from visualDet3D.data.kitti.kittidata import KittiData              # ImportError if the reference is not on sys.path

    def load(name):
        data_frame = KittiData(data_root_dir, name, output_dict)
        data_frame.calib, _, _, _ = data_frame.read_data()
        return data_frame

    print("start reading {} data".format(data_split))
    with ThreadPoolExecutor(WORKERS) as pool:
        frames = list(pool.map(load, index_names))
    save_dir = os.path.join(cfg.path.preprocessed_path, data_split)
    if not os.path.isdir(save_dir):
        os.makedirs(save_dir)
    with open(os.path.join(save_dir, 'imdb.pkl'), 'wb') as f:
        pickle.dump(frames, f)
    print("{} split finished precomputing".format(data_split))


def parse_args(argv=None):
    ap = argparse.ArgumentParser(prog="python -m visualdet3d_b200.det_precompute",
                                 description="The reference's det_precompute (imdb pickles and 3-D anchor priors), the priors on the GPU.")
    ap.add_argument("--config", default="config/config.py", help="the reference's config file (.py)")
    ap.add_argument("--split", default="train", choices=("train", "test"),
                    help="train: the training and validation pickles and the anchor priors; test: the test pickle")
    args = ap.parse_args(argv)
    if not args.config.endswith(".py"):
        ap.error(f"--config must name a .py config file, got {args.config!r}")
    return args


def main(config: str = "config/config.py", split: str = "train"):
    from visualDet3D.utils.utils import cfg_from_file                # ImportError if the reference is not on sys.path
    cfg = cfg_from_file(config)
    if split == "test":
        root = cfg.path.test_path
        names = ["%06d" % i for i in range(len(os.listdir(os.path.join(root, 'calib'))))]
        read_test_split(cfg, names, root, {"calib": True, "image": False, "label": False, "velodyne": False}, 'test', 100)
    else:
        if getattr(cfg, 'anchor_prior', True):
            torch.cuda.set_device(cfg.trainer.gpu)
        train_names, val_names = process_train_val_file(cfg)
        read_one_split(cfg, train_names, cfg.path.data_path, {"calib": True, "image": True, "label": True, "velodyne": False}, 'training', 100)
        read_one_split(cfg, val_names, cfg.path.data_path, {"calib": True, "image": False, "label": True, "velodyne": False}, 'validation',
                       100)
    print("Preprocessing finished")


if __name__ == "__main__":
    a = parse_args(sys.argv[1:])
    main(a.config, a.split)
