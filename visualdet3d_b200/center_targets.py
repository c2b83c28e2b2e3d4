"""KM3D and MonoFlex training targets on the GPU: the reference's `KittiRTM3DDataset._build_target` and
`KittiMonoFlexDataset._build_target` (R/data/kitti/dataset/KM3D_dataset.py:57-221, 346-527) with the heatmap splats, the keypoint
projection and the gathered regression targets computed by csrc/center_targets.cu.

`DeferredTargets.build(image_shape, P2, labels, ...)` packs one image's labels into a small record where `_build_target` ran (a DataLoader
worker).  `DeferredTargetBatch(targets)` stacks a batch's records into one staging buffer (what the collate_fn of
`plugin.install_train_targets_into_reference()` hands the training step); `.to_device()` uploads it, launches twice and returns the
reference's target dict (same keys, dtypes and [B, ...] shapes) as CUDA tensors.  `build_targets_host(targets)` computes the same dict with
the host form of the kernels' routines (the parity checker)."""
from __future__ import annotations

import ctypes
from typing import Dict, Sequence

import numpy as np
import torch

from . import _lib

MODE_KM3D, MODE_MONOFLEX = 0, 1
MAX_OBJECTS = 32
SCALE = 4
NUM_VERTEXES = {MODE_KM3D: 9, MODE_MONOFLEX: 10}

# The kernels' output slots, in the ABI's order (include/vd3d_b200.h): key, dtype, per-image shape as a function of (C, K, hm_h, hm_w).
_SLOTS = (
    ("hm", np.float32, lambda C, K, h, w: (C, h, w)),
    ("hm_hp", np.float32, lambda C, K, h, w: (K, h, w)),
    ("hps", np.float32, lambda C, K, h, w: (MAX_OBJECTS, 2 * K)),
    ("reg", np.float32, lambda C, K, h, w: (MAX_OBJECTS, 2)),
    ("hp_offset", np.float32, lambda C, K, h, w: (MAX_OBJECTS * K, 2)),
    ("dim", np.float32, lambda C, K, h, w: (MAX_OBJECTS, 3)),
    ("rots", np.float32, lambda C, K, h, w: (MAX_OBJECTS, 2)),
    ("rotbin", np.int64, lambda C, K, h, w: (MAX_OBJECTS, 2)),
    ("rotres", np.float32, lambda C, K, h, w: (MAX_OBJECTS, 2)),
    ("dep", np.float32, lambda C, K, h, w: (MAX_OBJECTS, 1)),
    ("ind", np.int64, lambda C, K, h, w: (MAX_OBJECTS,)),
    ("hp_ind", np.int64, lambda C, K, h, w: (MAX_OBJECTS * K,)),
    ("reg_mask", np.uint8, lambda C, K, h, w: (MAX_OBJECTS,)),
    ("hps_mask", np.uint8, lambda C, K, h, w: (MAX_OBJECTS, 2 * K)),
    ("hp_mask", np.uint8, lambda C, K, h, w: (MAX_OBJECTS * K,)),
    ("wh", np.float32, lambda C, K, h, w: (MAX_OBJECTS, 2)),
    ("location", np.float32, lambda C, K, h, w: (MAX_OBJECTS, 3)),
    ("ori", np.float32, lambda C, K, h, w: (MAX_OBJECTS, 1)),
    ("kp_detph_mask", np.float32, lambda C, K, h, w: (MAX_OBJECTS, 3)),        # the reference's spelling
    ("bboxes2d", np.float32, lambda C, K, h, w: (MAX_OBJECTS, 4)),
    ("bboxes2d_target", np.float32, lambda C, K, h, w: (MAX_OBJECTS, 4)),
)
_MONOFLEX_ONLY = ("kp_detph_mask", "bboxes2d", "bboxes2d_target")

# The order of the reference's target dicts (KM3D_dataset.py:200-219, 502-525)
KEYS = {
    MODE_KM3D: ("hm", "hm_hp", "hps", "reg", "hp_offset", "dim", "rots", "rotbin", "rotres", "dep", "ind", "hp_ind", "reg_mask",
                "hps_mask", "hp_mask", "wh", "location", "ori"),
    MODE_MONOFLEX: ("hm", "hm_hp", "hps", "reg", "hp_offset", "dim", "rots", "rotbin", "rotres", "dep", "ind", "hp_ind", "reg_mask",
                    "hps_mask", "hp_mask", "kp_detph_mask", "wh", "bboxes2d", "bboxes2d_target", "location", "ori", "edge_indices"),
}


def _vp(a: np.ndarray):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


def _shapes(mode, num_classes, img_h, img_w):
    K, hm_h, hm_w = NUM_VERTEXES[mode], img_h // SCALE, img_w // SCALE
    return [(key, dt, shp(num_classes, K, hm_h, hm_w)) for key, dt, shp in _SLOTS]


def edge_indices(img_h: int, img_w: int) -> np.ndarray:
    """KittiMonoFlexDataset._get_edge_utils((img_h, img_w), 4) (KM3D_dataset.py:301-343): the heatmap border as int64 (x, y) rows,
    unique and sorted.  The reference unpacks the (H, W) it is given as (img_w, img_h), so x runs to H // 4 and y to W // 4."""
    x_max, y_max = img_h // SCALE, img_w // SCALE
    y = np.arange(0, y_max)
    edges = [np.stack((np.zeros(len(y)), y), 1)]
    x = np.arange(0, x_max)
    edges.append(np.stack((x, np.full(len(x), y_max)), 1))
    y = np.arange(y_max, 0, -1)
    edges.append(np.stack((np.full(len(y), x_max), y), 1))
    x = np.arange(x_max, -1, -1)
    edges.append(np.stack((x, np.zeros(len(x))), 1))
    return np.unique(np.concatenate([e.astype(np.int64) for e in edges], 0), axis=0)


_EDGE_CACHE: Dict[tuple, torch.Tensor] = {}


def _edge_indices_device(img_h, img_w, B, device) -> torch.Tensor:
    key = (img_h, img_w, str(device))
    e = _EDGE_CACHE.get(key)
    if e is None:
        e = _EDGE_CACHE[key] = torch.from_numpy(edge_indices(img_h, img_w)).to(device)
    return e.unsqueeze(0).expand(B, -1, -1)


class DeferredTargets:
    """One image's targets, not yet computed: the packed record (mode, image size, class count, P2 and up to 32 objects)."""
    __slots__ = ("record", "mode", "img_h", "img_w", "num_classes")

    def __init__(self, record: np.ndarray, mode: int, img_h: int, img_w: int, num_classes: int):
        self.record, self.mode, self.img_h, self.img_w, self.num_classes = record, mode, img_h, img_w, num_classes

    @classmethod
    def build(cls, image_shape, P2, labels, cls_ids, num_classes: int, mode: int) -> "DeferredTargets":
        """`image_shape`: the augmented image's (H, W, ...); `P2` the float64 [3, 4] calibration; `labels` the KittiObj-like objects
        (x, y, z, w, h, l, ry, bbox_l / t / r / b); `cls_ids` their class indices.  More than 32 objects raise IndexError, as the
        reference's `orientation[k]` does."""
        if len(labels) > MAX_OBJECTS:
            raise IndexError(f"{len(labels)} objects: the targets hold max_objects = {MAX_OBJECTS}")
        img_h, img_w = int(image_shape[0]), int(image_shape[1])
        objs = np.array([[o.x, o.y, o.z, o.w, o.h, o.l, o.ry, o.bbox_l, o.bbox_t, o.bbox_r, o.bbox_b] for o in labels],
                        dtype=np.float64).reshape(-1, 11)
        ids = np.ascontiguousarray(cls_ids, dtype=np.int32).reshape(-1)
        p2 = np.ascontiguousarray(P2, dtype=np.float64).reshape(3, 4)
        rec = np.zeros(int(_lib.load().vd3d_center_targets_record_bytes()), dtype=np.uint8)
        _lib.call("vd3d_center_targets_pack", _vp(rec), mode, img_h, img_w, num_classes, _vp(p2), len(labels), _vp(objs), _vp(ids))
        return cls(rec, mode, img_h, img_w, num_classes)


def build_targets_host(t: DeferredTargets) -> Dict[str, np.ndarray]:
    """The reference's target dict of one image, computed on the host by the kernels' routines (the parity checker)."""
    outs = {key: np.zeros(shape, dt) for key, dt, shape in _shapes(t.mode, t.num_classes, t.img_h, t.img_w)
            if t.mode == MODE_MONOFLEX or key not in _MONOFLEX_ONLY}
    ptrs = (ctypes.c_void_p * len(_SLOTS))(*[outs[key].ctypes.data if key in outs else None for key, _, _ in _SLOTS])
    _lib.call("vd3d_center_targets_host", _vp(t.record), t.mode, t.img_h, t.img_w, t.num_classes, ptrs)
    if t.mode == MODE_MONOFLEX:
        outs["edge_indices"] = edge_indices(t.img_h, t.img_w)
    return {key: outs[key] for key in KEYS[t.mode]}


class DeferredTargetBatch:
    """The targets of one collated batch, not yet computed: the images' records in one staging buffer.  Built where the batch is collated
    (a DataLoader worker); `to_device` uploads it and runs the two launches."""

    def __init__(self, targets: Sequence[DeferredTargets]):
        assert len(targets) > 0
        t0 = targets[0]
        self.mode, self.img_h, self.img_w, self.num_classes = t0.mode, t0.img_h, t0.img_w, t0.num_classes
        for t in targets:
            assert (t.mode, t.img_h, t.img_w, t.num_classes) == (self.mode, self.img_h, self.img_w, self.num_classes), \
                "one detector, image size and class count per batch"
        nbytes = t0.record.nbytes
        self.staging = torch.empty(len(targets) * nbytes, dtype=torch.uint8)
        self.staging.numpy().reshape(len(targets), nbytes)[:] = np.stack([t.record for t in targets])

    def __len__(self):
        return self.staging.numel() // int(_lib.load().vd3d_center_targets_record_bytes())

    def pin_memory(self):
        self.staging = self.staging.pin_memory()
        return self

    def to_device(self, device="cuda") -> Dict[str, torch.Tensor]:
        """The reference's collated target dict ([B, ...] tensors of its dtypes) on `device`: one upload, two launches."""
        B = len(self)
        recs = self.staging.to(device, non_blocking=True)
        outs = {key: torch.empty((B,) + shape, dtype=getattr(torch, np.dtype(dt).name), device=device)
                for key, dt, shape in _shapes(self.mode, self.num_classes, self.img_h, self.img_w)
                if self.mode == MODE_MONOFLEX or key not in _MONOFLEX_ONLY}
        splats = torch.empty(B * int(_lib.load().vd3d_center_targets_splat_bytes()), dtype=torch.uint8, device=device)
        ptrs = (ctypes.c_void_p * len(_SLOTS))(*[outs[key].data_ptr() if key in outs else None for key, _, _ in _SLOTS])
        _lib.call("vd3d_center_targets", recs.data_ptr(), B, self.mode, self.img_h, self.img_w, self.num_classes, ptrs,
                  splats.data_ptr(), torch.cuda.current_stream(device).cuda_stream)
        outs["hm"]._vd3d_keepalive = (self.staging, recs, splats)     # must outlive the asynchronous copy and kernels
        if self.mode == MODE_MONOFLEX:
            outs["edge_indices"] = _edge_indices_device(self.img_h, self.img_w, B, device)
        return {key: outs[key] for key in KEYS[self.mode]}
