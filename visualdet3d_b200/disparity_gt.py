"""Stereo3D's disparity ground truth on the GPU (csrc/disparity_gt.cu): the two maps the reference's disparity precompute
(scripts/disparity_compute.py) writes for `DisparityLoss`, equal to its files in the decoded arrays.

    stereo_bm(left, right)                        cv2.StereoBM_create(192, 25).compute on uint8 grey [B, H, W] frames -> int16 [B, H, W]
    bm_targets(left_img, right_img, mean, std)    the script's StereoBM path from the test augmentation's float32 [B, H, W, 3] frames:
                                                  denorm, COLOR_BGR2GRAY, StereoBM, negatives to 0, 4x4 block max -> uint16 [B, H/4, W/4]
    velo_disparity(points, R0_rect, Tr_velo_to_cam, P2, baseline, H, W)
                                                  generate_dispariy_from_velo for one frame -> uint16 [H, W]
    velo_targets(...)                             the script's LiDAR path: velo_disparity, then the 4x4 block max -> uint16 [H/4, W/4]
    block_max(disp)                               skimage.measure.block_reduce(max(disp, 0), (4, 4), np.max) on [B, H, W] int16 / uint16

Every device function takes CUDA tensors, launches on the current stream and returns without synchronising; shapes, dtypes and devices
are checked before any launch.  The `*_host` functions compute the same maps on the host with the kernels' per-element routines (the
parity checker).  Heights below 26 and widths below 216 raise: cv2 has no defined StereoBM(192, 25) output there."""
from __future__ import annotations

import ctypes
from typing import Tuple

import numpy as np
import torch

from . import _lib

ND = 192
MIN_H, MIN_W = 26, 216
MAX_DIM = 1 << 14


def _vp(a: np.ndarray):
    return a.ctypes.data_as(ctypes.c_void_p)


def _stream(t: torch.Tensor) -> int:
    return torch.cuda.current_stream(t.device).cuda_stream


def _check_bm_shape(H: int, W: int) -> None:
    if not (MIN_H <= H <= MAX_DIM and MIN_W <= W <= MAX_DIM):
        raise ValueError(f"{H}x{W} frame: StereoBM(192, 25) needs {MIN_H} <= H and {MIN_W} <= W (and both <= {MAX_DIM})")


def _check_pair(left: torch.Tensor, right: torch.Tensor, dtype: torch.dtype, ndim: int) -> None:
    for name, t in (("left", left), ("right", right)):
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise ValueError(f"{name} must be a CUDA tensor")
        if t.dtype != dtype:
            raise TypeError(f"{name} must be {dtype}, got {t.dtype}")
        if t.dim() != ndim or (ndim == 4 and t.shape[-1] != 3):
            raise ValueError(f"{name} must be {'[B, H, W, 3]' if ndim == 4 else '[B, H, W]'}, got {list(t.shape)}")
    if left.shape != right.shape:
        raise ValueError(f"left {list(left.shape)} and right {list(right.shape)} differ")
    if left.device != right.device:
        raise ValueError(f"left on {left.device}, right on {right.device}")
    if left.shape[0] < 1 or left.shape[0] > 65535:
        raise ValueError(f"batch {left.shape[0]} outside [1, 65535]")
    _check_bm_shape(left.shape[1], left.shape[2])


def _workspace(B: int, H: int, W: int, device) -> torch.Tensor:
    n = int(_lib.load().vd3d_stereo_bm_workspace_bytes(B, H, W))
    if n < 0:
        raise _lib.Vd3dError(_lib.load().vd3d_last_error().decode())
    return torch.empty(n, dtype=torch.uint8, device=device)


def stereo_bm(left: torch.Tensor, right: torch.Tensor) -> torch.Tensor:
    """cv2.StereoBM_create(192, 25).compute(left[b], right[b]) for every frame: int16 [B, H, W], 16 x the disparity, -16 = filtered."""
    _check_pair(left, right, torch.uint8, 3)
    left, right = left.contiguous(), right.contiguous()
    B, H, W = left.shape
    ws = _workspace(B, H, W, left.device)
    disp = torch.empty((B, H, W), dtype=torch.int16, device=left.device)
    _lib.call("vd3d_stereo_bm", left.data_ptr(), right.data_ptr(), B, H, W, ws.data_ptr(), disp.data_ptr(), _stream(left))
    return disp


def _mean_std(mean, std) -> Tuple[np.ndarray, np.ndarray]:
    m = np.ascontiguousarray(mean, dtype=np.float64).reshape(-1)
    s = np.ascontiguousarray(std, dtype=np.float64).reshape(-1)
    if m.shape != (3,) or s.shape != (3,):
        raise ValueError(f"mean and std must hold 3 values each, got {m.shape} and {s.shape}")
    return m, s


def bm_disparity(left_img: torch.Tensor, right_img: torch.Tensor, mean, std, return_grey: bool = False):
    """StereoBM on the script's grey frames, from the normalised float32 [B, H, W, 3] network input: int16 [B, H, W].  With
    `return_grey`, also the uint8 grey frames [2, B, H, W] (left, then right) the matcher saw."""
    _check_pair(left_img, right_img, torch.float32, 4)
    left_img, right_img = left_img.contiguous(), right_img.contiguous()
    m, s = _mean_std(mean, std)
    B, H, W, _ = left_img.shape
    ws = _workspace(B, H, W, left_img.device)
    disp = torch.empty((B, H, W), dtype=torch.int16, device=left_img.device)
    grey = torch.empty((2, B, H, W), dtype=torch.uint8, device=left_img.device) if return_grey else None
    _lib.call("vd3d_stereo_bm_f32", left_img.data_ptr(), right_img.data_ptr(), B, H, W, _vp(m), _vp(s), ws.data_ptr(),
              grey.data_ptr() if grey is not None else None, disp.data_ptr(), _stream(left_img))
    return (disp, grey) if return_grey else disp


def block_max(disp: torch.Tensor) -> torch.Tensor:
    """The 4x4 block max of max(disp, 0) as uint16, far edges zero-padded: [B, ceil(H/4), ceil(W/4)] from int16 / uint16 [B, H, W]."""
    if not isinstance(disp, torch.Tensor) or not disp.is_cuda:
        raise ValueError("disp must be a CUDA tensor")
    if disp.dtype not in (torch.int16, torch.uint16):
        raise TypeError(f"disp must be int16 or uint16, got {disp.dtype}")
    if disp.dim() != 3 or min(disp.shape) < 1 or disp.shape[0] > 65535 or max(disp.shape[1:]) > MAX_DIM:
        raise ValueError(f"disp must be [B, H, W] with B <= 65535 and H, W <= {MAX_DIM}, got {list(disp.shape)}")
    disp = disp.contiguous()
    B, H, W = disp.shape
    out = torch.empty((B, -(-H // 4), -(-W // 4)), dtype=torch.uint16, device=disp.device)
    _lib.call("vd3d_disparity_block_max", disp.data_ptr(), int(disp.dtype == torch.int16), B, H, W, out.data_ptr(), _stream(disp))
    return out


def bm_targets(left_img: torch.Tensor, right_img: torch.Tensor, mean, std) -> torch.Tensor:
    """The map the precompute script writes on its StereoBM path, for every frame of the batch: uint16 [B, ceil(H/4), ceil(W/4)]."""
    return block_max(bm_disparity(left_img, right_img, mean, std))


def _calib(R0_rect, Tr_velo_to_cam, P2):
    R0 = np.ascontiguousarray(R0_rect, dtype=np.float64)
    Tr = np.ascontiguousarray(Tr_velo_to_cam, dtype=np.float64)
    p2 = np.ascontiguousarray(P2, dtype=np.float64)
    if R0.shape != (4, 4) or Tr.shape != (4, 4) or p2.shape != (3, 4):
        raise ValueError(f"R0_rect and Tr_velo_to_cam must be 4x4 and P2 3x4 (KittiCalib's), got {R0.shape}, {Tr.shape}, {p2.shape}")
    return R0, Tr, p2


def _check_hw(H: int, W: int) -> None:
    if not (1 <= H <= MAX_DIM and 1 <= W <= MAX_DIM):
        raise ValueError(f"{H}x{W} map outside [1, {MAX_DIM}]")


def velo_disparity(points: torch.Tensor, R0_rect, Tr_velo_to_cam, P2, baseline: float, H: int, W: int) -> torch.Tensor:
    """generate_dispariy_from_velo(points[:, :3], H, W, Tr_velo_to_cam, R0_rect, P2, baseline): uint16 [H, W], the last in-view point of
    each pixel in cloud order, 0 where none.  points: float32 [N, C >= 3] CUDA (a KITTI scan's [N, 4]); the calibration as numpy."""
    if not isinstance(points, torch.Tensor) or not points.is_cuda:
        raise ValueError("points must be a CUDA tensor")
    if points.dtype != torch.float32:
        raise TypeError(f"points must be float32, got {points.dtype}")
    if points.dim() != 2 or points.shape[1] < 3 or points.shape[0] >= 2 ** 31:
        raise ValueError(f"points must be [N, C] with C >= 3, got {list(points.shape)}")
    R0, Tr, p2 = _calib(R0_rect, Tr_velo_to_cam, P2)
    H, W = int(H), int(W)
    _check_hw(H, W)
    points = points.contiguous()
    winner = torch.empty((H, W), dtype=torch.int32, device=points.device)
    full = torch.empty((H, W), dtype=torch.uint16, device=points.device)
    _lib.call("vd3d_velo_disparity", points.data_ptr(), points.shape[0], points.shape[1], _vp(R0), _vp(Tr), _vp(p2), float(baseline), H, W,
              winner.data_ptr(), full.data_ptr(), _stream(points))
    return full


def velo_targets(points: torch.Tensor, R0_rect, Tr_velo_to_cam, P2, baseline: float, H: int, W: int) -> torch.Tensor:
    """The map the precompute script writes on its LiDAR path: uint16 [ceil(H/4), ceil(W/4)]."""
    return block_max(velo_disparity(points, R0_rect, Tr_velo_to_cam, P2, baseline, H, W)[None])[0]


# ---- host forms (the parity checker) -----------------------------------------------------------------------------------------------

def grey_host(img: np.ndarray, mean, std) -> np.ndarray:
    """cv2.cvtColor(denorm(img, mean, std), COLOR_BGR2GRAY) of one float32 [H, W, 3] frame: uint8 [H, W]."""
    img = np.ascontiguousarray(img, dtype=np.float32)
    if img.ndim != 3 or img.shape[2] != 3:
        raise ValueError(f"img must be [H, W, 3], got {img.shape}")
    m, s = _mean_std(mean, std)
    out = np.empty(img.shape[:2], np.uint8)
    _lib.call("vd3d_disparity_grey_host", _vp(img), img.shape[0], img.shape[1], _vp(m), _vp(s), _vp(out))
    return out


def stereo_bm_host(left: np.ndarray, right: np.ndarray) -> np.ndarray:
    """stereo_bm of one uint8 [H, W] pair on the host: int16 [H, W]."""
    left, right = np.ascontiguousarray(left, np.uint8), np.ascontiguousarray(right, np.uint8)
    if left.ndim != 2 or left.shape != right.shape:
        raise ValueError(f"left {left.shape} and right {right.shape} must be equal [H, W]")
    _check_bm_shape(*left.shape)
    out = np.empty(left.shape, np.int16)
    _lib.call("vd3d_stereo_bm_host", _vp(left), _vp(right), left.shape[0], left.shape[1], _vp(out))
    return out


def block_max_host(disp: np.ndarray) -> np.ndarray:
    disp = np.ascontiguousarray(disp)
    if disp.dtype not in (np.int16, np.uint16) or disp.ndim != 2:
        raise ValueError(f"disp must be int16 or uint16 [H, W], got {disp.dtype} {disp.shape}")
    H, W = disp.shape
    out = np.empty((-(-H // 4), -(-W // 4)), np.uint16)
    _lib.call("vd3d_disparity_block_max_host", _vp(disp), int(disp.dtype == np.int16), H, W, _vp(out))
    return out


def velo_disparity_host(points: np.ndarray, R0_rect, Tr_velo_to_cam, P2, baseline: float, H: int, W: int) -> np.ndarray:
    pts = np.ascontiguousarray(points, np.float32)
    if pts.ndim != 2 or pts.shape[1] < 3:
        raise ValueError(f"points must be [N, C] with C >= 3, got {pts.shape}")
    R0, Tr, p2 = _calib(R0_rect, Tr_velo_to_cam, P2)
    _check_hw(int(H), int(W))
    out = np.empty((int(H), int(W)), np.uint16)
    _lib.call("vd3d_velo_disparity_host", _vp(pts), pts.shape[0], pts.shape[1], _vp(R0), _vp(Tr), _vp(p2), float(baseline), int(H), int(W),
              _vp(out))
    return out
