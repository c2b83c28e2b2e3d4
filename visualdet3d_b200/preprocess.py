"""Test-time input pipeline (SURVEY.md section 8(f) rank 3): what the reference's `test_augmentation` does per frame on the CPU with cv2 /
numpy (R/data/pipeline/stereo_augmentator.py: ConvertToFloat :29-36, CropTop :213-258, Resize :63-134, Normalize :39-60) and
`KittiStereoDataset.__getitem__` / `collate_fn` (R/data/kitti/dataset/stereo_dataset.py:176-203): uint8 HWC frame -> float32 CHW network
input, and the calibration matrices moved along.

The image work is the training augmentation's geometry 0 with no photometric program and no mirror: `preprocess_host` / `preprocess_batch`
are `train_augment.augment_host` / `augment_batch` on such DeferredFrames (one per-pixel routine shared by the host entry and the CUDA
kernel).  The calibration update is host float arithmetic in the reference's order."""
from __future__ import annotations

from typing import List, Tuple

import numpy as np
import torch

from . import train_augment as ta

RGB_MEAN = (0.485, 0.456, 0.406)
RGB_STD = (0.229, 0.224, 0.225)

# The augmentation parameters of the test-time pipeline: CropTop + Resize, no warp, no mirror, no photometric program.
RESIZE_ONLY = dict(geom=ta.GEOM_RESIZE, affine=np.zeros((2, 3), np.float32), mirror=0, ops=np.zeros(0, np.int32), args=np.zeros(0, np.float32),
                   noise=np.zeros(3))


def adjust_calib(P: np.ndarray, crop_top: int, height: int, out_height: int) -> np.ndarray:
    """P [3, 4] of the original frame -> P of the network input: CropTop (cy -= dv, ty -= dv * tz) then Resize (rows 0 and 1 scaled)."""
    P = np.array(P, copy=True)
    P[1, 2] = P[1, 2] - crop_top
    P[1, 3] = P[1, 3] - crop_top * P[2, 3]
    s = out_height / (height - crop_top)
    P[0, :] = P[0, :] * s
    P[1, :] = P[1, :] * s
    return P


def _deferred(frame: np.ndarray, crop_top: int, size: Tuple[int, int], mean, std) -> ta.DeferredFrame:
    return ta.DeferredFrame(frame, crop_top=int(crop_top), Ho=int(size[0]), Wo=int(size[1]), mean=mean, std=std, **RESIZE_ONLY)


def preprocess_host(frame: np.ndarray, crop_top: int, size: Tuple[int, int], mean=RGB_MEAN, std=RGB_STD) -> np.ndarray:
    """uint8 [H, W, 3] -> float32 [3, size[0], size[1]] on the host: the parity checker of the CUDA form (`preprocess_batch` is the product
    path; tests pin this routine to the reference and the kernel to this routine)."""
    return ta.augment_host(_deferred(frame, crop_top, size, mean, std))


def preprocess_batch(frames: List[np.ndarray], crop_top: int, size: Tuple[int, int], mean=RGB_MEAN, std=RGB_STD, device="cuda") -> torch.Tensor:
    """uint8 HWC frames (sizes may differ) -> [B, 3, size[0], size[1]] float32 on `device`: one upload of the uint8 frames (3 bytes per pixel
    instead of 12) and one kernel for the whole batch."""
    return ta.augment_batch([_deferred(f, crop_top, size, mean, std) for f in frames], device)
