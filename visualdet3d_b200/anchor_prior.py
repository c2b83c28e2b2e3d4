"""The 3-D anchor priors of the reference's det_precompute (scripts/imdb_precompute_3d.py: read_one_split) on the GPU
(csrc/anchor_prior.cu): `anchor_{mean,std}_{type}.npy`, the per-(scale, ratio) (z, sin 2a, cos 2a, w, h, l) statistics the 3-D anchor
detectors read when they are built (`anchors.load_priors`).

    AnchorPriorAccumulator(anchors_cfg, image_hw, obj_types, fg_iou_threshold, device)
        .count_objects(labels)      the split-wide class statistics of one frame's (unaugmented, filtered) labels
        .add(frames, image_hw)      one batch: each frame's labels after the test augmentation; launches, does not synchronise
        .finalize()                 per class (mean, std) float64 [rows, ratios, 6], the reference's host formula, sentinels included
    accumulate(state, ...)          the device entry on packed tensors; accumulate_host(...) the same on numpy arrays (the parity checker)
    bin_table32(anchors32, ...)     the reference's anchors2indexes on the float32 table, as the script calls it

Exactness, from the reference's code:
  - the IoU's dtype is torch.tensor's inference on the label values: python floats (every shipped test list) give float32, numpy float64
    values (a Resize whose size is a numpy array) give float64; the threshold is compared in that dtype (0.6 != 0.6f).
  - (z, sin 2a, cos 2a) is float64 (np.sin makes the row float64), squares too.
  - the bin of a positive comes from the float32 anchors (`used_anchors` is a float32 .cpu().numpy()), unlike `anchors.prior_lookup`,
    which works on the float64 table."""
from __future__ import annotations

import ctypes
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .anchors import grid_anchors

MAX_K = 512                 # boxes per (frame, class) segment
MAX_SEGMENTS = 65535        # frames x classes per launch (the grid's y limit) ...
MAX_FLAG_BYTES = 1 << 30    # ... and at most this much positive-box workspace, [segments, anchors] int32


def _vp(a: np.ndarray):
    return a.ctypes.data_as(ctypes.c_void_p)


def bin_table32(anchors32: np.ndarray, sizes, ratios, scales) -> Tuple[np.ndarray, np.ndarray]:
    """(size row, ratio column) of each float32 anchor: Anchors.anchors2indexes (R/networks/heads/anchors.py:45-57) verbatim, so sqrt(w*h)
    and h/w round in float32 and the float64 grids are subtracted after."""
    sizes_ = np.sqrt((anchors32[:, 2] - anchors32[:, 0]) * (anchors32[:, 3] - anchors32[:, 1]))
    sizes_diff = sizes_ - (np.array(sizes) * np.array(scales))[:, np.newaxis]
    sizes_int = np.argmin(np.abs(sizes_diff), axis=0)
    ratio = (anchors32[:, 3] - anchors32[:, 1]) / (anchors32[:, 2] - anchors32[:, 0])
    ratio_diff = ratio - np.array(ratios)[:, np.newaxis]
    ratio_int = np.argmin(np.abs(ratio_diff), axis=0)
    return sizes_int, ratio_int


def bin_order(bins: np.ndarray, n_bins: int) -> Tuple[np.ndarray, np.ndarray]:
    """The anchors of each bin in ascending index, and the bins' starts: (order [N] int32, bin_start [n_bins + 1] int32)."""
    bins = np.asarray(bins)
    if bins.ndim != 1 or (bins.size and (bins.min() < 0 or bins.max() >= n_bins)):
        raise ValueError(f"bins must be a 1-D array of values in [0, {n_bins})")
    order = np.argsort(bins, kind="stable").astype(np.int32)
    start = np.zeros(n_bins + 1, dtype=np.int32)
    start[1:] = np.cumsum(np.bincount(bins, minlength=n_bins))
    return order, start


class PriorState:
    """The accumulator state: examine [T, bins] int64, sums / squared [T, bins, 3] float64, usable [T] int64, on `device` (or numpy)."""

    def __init__(self, T: int, n_bins: int, device=None):
        if device is None:
            self.examine = np.zeros((T, n_bins), np.int64)
            self.sums = np.zeros((T, n_bins, 3))
            self.squared = np.zeros((T, n_bins, 3))
            self.usable = np.zeros(T, np.int64)
        else:
            self.examine = torch.zeros((T, n_bins), dtype=torch.int64, device=device)
            self.sums = torch.zeros((T, n_bins, 3), dtype=torch.float64, device=device)
            self.squared = torch.zeros((T, n_bins, 3), dtype=torch.float64, device=device)
            self.usable = torch.zeros(T, dtype=torch.int64, device=device)
        self.T, self.n_bins = T, n_bins

    def numpy(self) -> Dict[str, np.ndarray]:
        """The four arrays on the host (synchronises when they are on a device)."""
        f = (lambda a: a.cpu().numpy()) if isinstance(self.examine, torch.Tensor) else np.array
        return {k: f(getattr(self, k)) for k in ("examine", "sums", "squared", "usable")}


def _host_ints(a, name: str, n: int) -> np.ndarray:
    if isinstance(a, torch.Tensor):
        if a.is_cuda:
            raise ValueError(f"{name} must be on the host")
        a = a.numpy()
    a = np.asarray(a)
    if a.dtype.kind not in "iu" or a.shape != (n, ):
        raise ValueError(f"{name} must hold {n} integers, got {a.dtype} {list(a.shape)}")
    return np.ascontiguousarray(a, dtype=np.int32)


def _sizes(state: PriorState, N: int, order_n: int, bin_start, offsets, K: int):
    bs = _host_ints(bin_start, "bin_start", state.n_bins + 1)
    if isinstance(offsets, torch.Tensor):
        if offsets.is_cuda:
            raise ValueError("offsets must be on the host")
        offsets = offsets.numpy()
    off = np.asarray(offsets)
    if off.ndim != 1 or off.size < 2 or (off.size - 1) % state.T:
        raise ValueError(f"offsets must hold B * T + 1 values (T = {state.T}), got {list(off.shape)}")
    off = _host_ints(off, "offsets", off.size)
    if order_n != N:
        raise ValueError(f"order holds {order_n} anchors, the table {N}")
    if off[0] != 0 or off[-1] != K or np.any(np.diff(off) < 0) or np.any(np.diff(off) > MAX_K):
        raise ValueError(f"offsets must rise from 0 to the {K} boxes by at most {MAX_K} per segment")
    if bs[0] != 0 or bs[-1] != N or np.any(np.diff(bs) < 0):
        raise ValueError(f"bin_start must rise from 0 to N = {N}")
    return bs, off, (off.size - 1) // state.T


def accumulate(state: PriorState, anchors: torch.Tensor, order: torch.Tensor, bin_start, offsets, boxes: torch.Tensor, gt3: torch.Tensor,
               fg_iou_threshold: float) -> None:
    """One batch into the device state.  anchors [N, 4] float32, order [N] int32 (bin_order), boxes [K, 4] float32 or float64 (the IoU's
    dtype), gt3 [K, 3] float64: CUDA tensors on the state's device.  bin_start [bins + 1] and offsets [B*T + 1] (segment b * T + t):
    host integers.  Launches on the current stream without synchronising."""
    prepare(state, anchors, order, bin_start, offsets, boxes, gt3, fg_iou_threshold)()


def prepare(state: PriorState, anchors: torch.Tensor, order: torch.Tensor, bin_start, offsets, boxes: torch.Tensor, gt3: torch.Tensor,
            fg_iou_threshold: float):
    """`accumulate`'s checks and workspace; returns the call of the entry itself (offsets copy, key memset, two launches), so that a
    benchmark can time the launches apart from the Python around them.  Each call adds the batch once more."""
    dev = state.examine.device
    for name, t, dts, cols in (("anchors", anchors, (torch.float32, ), 4), ("order", order, (torch.int32, ), None),
                               ("boxes", boxes, (torch.float32, torch.float64), 4), ("gt3", gt3, (torch.float64, ), 3)):
        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.device != dev:
            raise ValueError(f"{name} must be a CUDA tensor on {dev}")
        if t.dtype not in dts:
            raise TypeError(f"{name} must be {' or '.join(str(d) for d in dts)}, got {t.dtype}")
        if (t.dim() != 1) if cols is None else (t.dim() != 2 or t.shape[1] != cols):
            raise ValueError(f"{name} has shape {list(t.shape)}")
    if boxes.shape[0] != gt3.shape[0]:
        raise ValueError(f"{boxes.shape[0]} boxes but {gt3.shape[0]} gt3 rows")
    N, K = anchors.shape[0], boxes.shape[0]
    bs, off, B = _sizes(state, N, order.shape[0], bin_start, offsets, K)
    if B * state.T > MAX_SEGMENTS or B * state.T * N * 4 > MAX_FLAG_BYTES:
        raise ValueError(f"{B} frames x {state.T} classes x {N} anchors: at most {MAX_SEGMENTS} segments and {MAX_FLAG_BYTES} bytes of "
                         f"positive-box workspace per launch ({max_frames_per_launch(N, state.T)} frames here)")
    lib = _lib.load()
    nbytes = int(lib.vd3d_anchor_prior_workspace_bytes(N, state.n_bins, B, state.T, K))
    if nbytes < 0:
        raise _lib.Vd3dError(lib.vd3d_last_error().decode())
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    anchors, order, boxes, gt3 = anchors.contiguous(), order.contiguous(), boxes.contiguous(), gt3.contiguous()
    args = (anchors.data_ptr(), order.data_ptr(), _vp(bs), N, state.n_bins, _vp(off), B, state.T, boxes.data_ptr(),
            int(boxes.dtype == torch.float64), gt3.data_ptr(), K, float(fg_iou_threshold), state.examine.data_ptr(), state.sums.data_ptr(),
            state.squared.data_ptr(), state.usable.data_ptr(), ws.data_ptr(), nbytes, torch.cuda.current_stream(dev).cuda_stream)
    keep = (anchors, order, boxes, gt3, ws, bs, off)                  # alive as long as the returned call

    def call():
        _lib.call("vd3d_anchor_prior_accumulate", *args)
        return keep
    return call


def accumulate_host(state: PriorState, anchors: np.ndarray, order: np.ndarray, bin_start, offsets, boxes: np.ndarray, gt3: np.ndarray,
                    fg_iou_threshold: float) -> None:
    """`accumulate` on numpy arrays and a host state, in the reference's loop order (vd3d_anchor_prior_host)."""
    anchors = np.ascontiguousarray(anchors, dtype=np.float32)
    order = np.ascontiguousarray(order, dtype=np.int32)
    if boxes.dtype not in (np.float32, np.float64):
        raise TypeError(f"boxes must be float32 or float64, got {boxes.dtype}")
    boxes = np.ascontiguousarray(boxes).reshape(-1, 4)
    gt3 = np.ascontiguousarray(gt3, dtype=np.float64).reshape(-1, 3)
    N, K = anchors.shape[0], boxes.shape[0]
    bs, off, B = _sizes(state, N, order.shape[0], bin_start, offsets, K)
    _lib.call("vd3d_anchor_prior_host", _vp(anchors), _vp(order), _vp(bs), N, state.n_bins, _vp(off), B, state.T, _vp(boxes),
              int(boxes.dtype == np.float64), _vp(gt3), K, float(fg_iou_threshold), _vp(state.examine), _vp(state.sums),
              _vp(state.squared), _vp(state.usable))


def _box_dtype(rows) -> torch.dtype:
    """torch.tensor(rows).dtype, the dtype of the script's box tensor and so of its IoU, without building the tensor when every value is
    a python float (float32)."""
    if all(type(v) is float for r in rows for v in r):
        return torch.float32
    dt = torch.tensor(rows).dtype
    if dt not in (torch.float32, torch.float64):
        raise TypeError(f"box values of dtype {dt}: the IoU is computed in float32 or float64 only")
    return dt


def max_frames_per_launch(N: int, T: int) -> int:
    """Frames per launch whose [segments, N] int32 positive-box workspace stays within MAX_FLAG_BYTES (and the grid's segment limit)."""
    return max(1, min(MAX_SEGMENTS, MAX_FLAG_BYTES // (4 * N)) // T)


class AnchorPriorAccumulator:
    """The anchor-prior half of read_one_split for one split, its per-frame IoU and statistics on `device`."""

    def __init__(self, anchors_cfg, image_hw, obj_types: Sequence[str], fg_iou_threshold: float, device="cuda", config_name: str = "config"):
        """device=None keeps the state on the host and accumulates with the host entry (the parity checker)."""
        self.cfg = anchors_cfg
        self.obj_types = list(obj_types)
        self.thr = float(fg_iou_threshold)
        self.device = None if device is None else torch.device(device)
        self.config_name = config_name
        self.rows = len(anchors_cfg["pyramid_levels"]) * len(anchors_cfg["scales"])
        self.ratios = len(anchors_cfg["ratios"])
        self.state = PriorState(len(self.obj_types), self.rows * self.ratios, self.device)
        self.total_objects = [0 for _ in self.obj_types]
        self.uniform_sum = np.zeros((len(self.obj_types), 6), dtype=np.float64)
        self.uniform_square = np.zeros((len(self.obj_types), 6), dtype=np.float64)
        self._tables = {}
        self.image_hw = None if image_hw is None else tuple(int(v) for v in image_hw)
        if self.image_hw is not None:
            self.table(self.image_hw)

    def table(self, image_hw):
        """(anchors [N, 4] float32, order, bin_start) for one post-augmentation shape, built once and kept on the device."""
        hw = tuple(int(v) for v in image_hw)
        if hw not in self._tables:
            c = self.cfg
            a32 = grid_anchors(hw, c["pyramid_levels"], c["strides"], c["sizes"], c["ratios"], c["scales"]).astype(np.float32)
            try:
                rows, cols = bin_table32(a32, c["sizes"], c["ratios"], c["scales"])
            except ValueError as e:
                raise ValueError(f"{self.config_name}: the reference's anchors2indexes cannot map this anchor config's "
                                 f"{len(c['sizes'])} sizes x {len(c['scales'])} scales onto prior rows ({e})") from None
            order, start = bin_order(rows * self.ratios + cols, self.rows * self.ratios)
            if self.device is None:
                self._tables[hw] = (a32, order, start)
            else:
                self._tables[hw] = (torch.from_numpy(a32).to(self.device), torch.from_numpy(order).to(self.device), start)
        return self._tables[hw]

    def count_objects(self, labels) -> None:
        """imdb_precompute_3d.py:83-93 for one frame: object counts and the (z, sin 2a, cos 2a, w, h, l) sums of each class."""
        for j, name in enumerate(self.obj_types):
            self.total_objects[j] += len([obj for obj in labels if obj.type == name])
            data = np.array([[obj.z, np.sin(2 * obj.alpha), np.cos(2 * obj.alpha), obj.w, obj.h, obj.l] for obj in labels if obj.type == name])
            if data.any():
                self.uniform_sum[j, :] += np.sum(data, axis=0)
                self.uniform_square[j, :] += np.sum(data ** 2, axis=0)

    def add(self, frames: List[list], image_hw=None) -> None:
        """One batch of frames (each a list of labels after the test augmentation, all of shape `image_hw`), accumulated in order.

        The script builds each (frame, class) box tensor on its own, so each segment has its own IoU dtype.  One launch takes one dtype:
        frames are grouped into runs in which every class keeps one dtype, and a run whose classes differ is launched once per dtype,
        with the other dtype's segments left empty.  A class's segments therefore always reach its bins in frame order."""
        T = len(self.obj_types)
        segs = []
        for labels in frames:
            for name in self.obj_types:
                objs = [obj for obj in labels if obj.type == name]
                if len(objs) > MAX_K:
                    raise ValueError(f"a frame holds {len(objs)} objects of class {name} (at most {MAX_K})")
                box = [[obj.bbox_l, obj.bbox_t, obj.bbox_r, obj.bbox_b] for obj in objs]
                segs.append((box, [[obj.z, np.sin(2 * obj.alpha), np.cos(2 * obj.alpha)] for obj in objs],
                             _box_dtype(box) if box else None))
        anchors, order, start = self.table(image_hw or self.image_hw)
        cap = max_frames_per_launch(anchors.shape[0], T)
        f0, nf = 0, len(frames)
        while f0 < nf:
            kind = [None] * T                                 # each class's dtype in this run
            f1 = f0
            while f1 < nf and f1 - f0 < cap:
                ds = [segs[f1 * T + t][2] for t in range(T)]
                if any(d is not None and kind[t] is not None and d != kind[t] for t, d in enumerate(ds)):
                    break
                kind = [k if d is None else d for k, d in zip(kind, ds)]
                f1 += 1
            for dt in sorted({d for d in kind if d is not None}, key=str):
                run = [sg if kind[i % T] == dt else ([], [], None) for i, sg in enumerate(segs[f0 * T:f1 * T])]
                self._launch(run, dt, anchors, order, start)
            f0 = f1

    def _launch(self, run, dt, anchors, order, start) -> None:
        off = np.zeros(len(run) + 1, dtype=np.int32)
        off[1:] = np.cumsum([len(b) for b, _, _ in run])
        boxes = torch.tensor([r for b, _, _ in run for r in b], dtype=dt)
        gt3 = torch.tensor([r for _, g, _ in run for r in g], dtype=torch.float64)
        if self.device is None:
            accumulate_host(self.state, anchors, order, start, off, boxes.numpy(), gt3.numpy(), self.thr)
        else:
            accumulate(self.state, anchors, order, start, off, boxes.pin_memory().to(self.device, non_blocking=True),
                       gt3.pin_memory().to(self.device, non_blocking=True), self.thr)

    def usable_objects(self) -> List[int]:
        return [int(v) for v in self.state.numpy()["usable"]]

    def finalize(self) -> List[Tuple[np.ndarray, np.ndarray]]:
        """Per class (mean, std), each float64 [rows, ratios, 6]: imdb_precompute_3d.py:150-169 on the accumulated state."""
        st = self.state.numpy()
        return priors_from_state(st, self.rows, self.ratios, self.uniform_sum, self.uniform_square, self.total_objects)


def priors_from_state(st: Dict[str, np.ndarray], rows: int, ratios: int, uniform_sum, uniform_square, total_objects):
    """imdb_precompute_3d.py:150-169: per class (mean, std) from the accumulator state (PriorState.numpy()) and the split-wide class
    sums, with the script's sentinels (-100 / 1e10 where examine < 10, std is NaN or std < 1e-3) and, for a class with no object,
    its NaN w / h / l columns."""
    T = len(total_objects)
    examine = st["examine"].astype(np.float64).reshape(T, rows, ratios)
    sums = st["sums"].reshape(T, rows, ratios, 3)
    squared = st["squared"].reshape(T, rows, ratios, 3)
    out = []
    for j in range(T):
        global_mean = uniform_sum[j] / total_objects[j]
        global_var = np.sqrt(uniform_square[j] / total_objects[j] - global_mean ** 2)

        avg = sums[j] / (examine[j][:, :, np.newaxis] + 1e-8)
        EX_2 = squared[j] / (examine[j][:, :, np.newaxis] + 1e-8)
        std = np.sqrt(EX_2 - avg ** 2)

        avg[examine[j] < 10, :] = -100
        std[examine[j] < 10, :] = 1e10
        avg[np.isnan(std)] = -100
        std[np.isnan(std)] = 1e10
        avg[std < 1e-3] = -100
        std[std < 1e-3] = 1e10

        whl_avg = np.ones([avg.shape[0], avg.shape[1], 3]) * global_mean[3:6]
        whl_std = np.ones([avg.shape[0], avg.shape[1], 3]) * global_var[3:6]
        out.append((np.concatenate([avg, whl_avg], axis=2), np.concatenate([std, whl_std], axis=2)))
    return out
