"""Training loss of the RetinaNet head on the GPU: the reference's `RetinanetHead.loss` (R/networks/heads/retinanet_head.py:309-362;
R/ = visualDet3D in the reference tree), as one autograd Function over csrc/retina_loss.cu.

The anchor assignment (calc_iou, _assign with low-quality matching), the one-hot sigmoid focal terms, _encode, the _decode of the
prediction and of the encoded target, the IoU loss and the batch reduction run in four launches with no host synchronisation; the
backward is one launch.  Sums are reduced in a fixed order without float atomics, so two runs give the same bits and the pair can be
captured in a CUDA graph.  There is no CPU path.

Two inputs where the native loss departs from the reference:
  * no positive anchor in the whole batch: the reference's reg_loss stays the Python number 0 / 1e-4 (and train_mono_detection's
    `.mean()` on it then raises); here it is a 0-d tensor 0 whose gradient is zero;
  * a positive anchor whose ground truth's class.long() lies outside [0, C): the reference's label scatter fails from C up and below
    -C, and wraps -C..-1 (class -1 is padding, but e.g. -2 or -1.5 is not) into column C + class, labelling another class; here both
    losses and every gradient are NaN in all these cases, without a host synchronisation.

    retinanet_head_loss(cls_scores, reg_preds, anchors, annotations, cfg)  -> (cls_loss 0-d, reg_loss 0-d, loss dict)
    assignment(...)                                                        -> (assigned_gt_inds [B, N] i32, counts [B, 3] i32)
    head_loss                                                              the method `plugin.install_retinanet_loss_into_reference()` binds
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Mapping, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .loss_common import as_config, cached_on, check, grad_out_pair, stream, workspace

MAX_CLASSES = 64
MAX_ROWS = 512          # annotation rows per image the kernels hold in shared memory
ANN_COLS = 5            # x1 y1 x2 y2 class: the annotation columns the loss reads


@dataclass(frozen=True)
class LossConfig:
    """The settings the reference's loss reads, with `_assign` / `build_loss` / `RetinanetHead` defaults (retinanet_head.py:15-25, 73-104)."""
    num_classes: int
    fg_iou_threshold: float = 0.5
    bg_iou_threshold: float = 0.0
    min_iou_threshold: float = 0.0
    match_low_quality: bool = True
    gt_max_assign_all: bool = True
    gamma: float = 0.0
    balance_weights: Tuple[float, ...] = (0.0,)
    target_means: Tuple[float, ...] = (0.0, 0.0, 0.0, 0.0)
    target_stds: Tuple[float, ...] = (1.0, 1.0, 1.0, 1.0)

    def __post_init__(self):
        if not 1 <= self.num_classes <= MAX_CLASSES:
            raise ValueError(f"retina loss: num_classes must be in 1..{MAX_CLASSES}, got {self.num_classes}")
        if len(self.balance_weights) not in (1, self.num_classes):
            raise ValueError(f"retina loss: balance_weights has {len(self.balance_weights)} entries; it needs 1 or num_classes "
                             f"({self.num_classes})")
        if len(self.target_means) != 4 or len(self.target_stds) != 4:
            raise ValueError(f"retina loss: target_means / target_stds need 4 entries, got {len(self.target_means)} / "
                             f"{len(self.target_stds)}")

    @classmethod
    def from_loss_cfg(cls, loss_cfg: Mapping, num_classes: int, target_means: Sequence[float] = (0.0, 0.0, 0.0, 0.0),
                      target_stds: Sequence[float] = (1.0, 1.0, 1.0, 1.0)) -> "LossConfig":
        """From a config's `detector.head.loss_cfg` (R/config/RetinaNet_example: head_loss) and the head's target_means / target_stds."""
        get = loss_cfg.get
        return cls(num_classes=int(num_classes),
                   fg_iou_threshold=float(get("fg_iou_threshold", 0.5)),
                   bg_iou_threshold=float(get("bg_iou_threshold", 0.0)),
                   min_iou_threshold=float(get("min_iou_threshold", 0.0)),
                   match_low_quality=bool(get("match_low_quality", True)),
                   gt_max_assign_all=bool(get("gt_max_assign_all", True)),
                   gamma=float(get("gamma", 0.0)),
                   balance_weights=tuple(float(v) for v in np.asarray(get("balance_weights", 0), dtype=np.float32).reshape(-1)),
                   target_means=tuple(float(v) for v in target_means),
                   target_stds=tuple(float(v) for v in target_stds))

    @classmethod
    def from_head(cls, head) -> "LossConfig":
        """From a reference RetinanetHead's own attributes: num_clasess (sic), loss_cfg, target_means / target_stds, and the focal loss
        it calls (loss_cls.gamma and its balance_weights buffer, a copy of the head's)."""
        lc = head.loss_cfg
        return cls(num_classes=int(head.num_clasess),
                   fg_iou_threshold=float(lc.get("fg_iou_threshold", 0.5)),
                   bg_iou_threshold=float(lc.get("bg_iou_threshold", 0.0)),
                   min_iou_threshold=float(lc.get("min_iou_threshold", 0.0)),
                   match_low_quality=bool(lc.get("match_low_quality", True)),
                   gt_max_assign_all=bool(lc.get("gt_max_assign_all", True)),
                   gamma=float(head.loss_cls.gamma),
                   balance_weights=tuple(float(v) for v in head.loss_cls.balance_weights.reshape(-1).tolist()),
                   target_means=tuple(float(v) for v in head.target_means),
                   target_stds=tuple(float(v) for v in head.target_stds))

    def params(self) -> np.ndarray:
        """The float32 parameter block of vd3d_retina_loss_forward / _backward (include/vd3d_b200.h)."""
        bw = self.balance_weights * (self.num_classes if len(self.balance_weights) == 1 else 1)
        return np.ascontiguousarray(np.array([self.fg_iou_threshold, self.bg_iou_threshold, self.min_iou_threshold, self.gamma,
                                              *self.target_means, *self.target_stds, *bw], dtype=np.float32))


def _inputs(cls_scores, reg_preds, anchors, annotations, cfg: LossConfig):
    """Host-side checks of what the kernels require, before any launch."""
    if cls_scores.dim() != 3:
        raise ValueError(f"retina loss: cls_scores {tuple(cls_scores.shape)}, expected [B, N, C]")
    B, N, C = cls_scores.shape
    if C != cfg.num_classes:
        raise ValueError(f"retina loss: cls_scores has {C} columns, the head {cfg.num_classes} classes")
    if tuple(reg_preds.shape) != (B, N, 4):
        raise ValueError(f"retina loss: reg_preds {tuple(reg_preds.shape)}, expected {(B, N, 4)}")
    anchor = anchors[0] if anchors.dim() == 3 else anchors          # get_anchor's [1, N, 4]; the reference reads anchors[0]
    if tuple(anchor.shape) != (N, 4):
        raise ValueError(f"retina loss: anchors {tuple(anchors.shape)} do not hold the {N} boxes of cls_scores")
    if annotations.dim() != 3 or annotations.shape[0] != B or annotations.shape[2] < ANN_COLS:
        raise ValueError(f"retina loss: annotations {tuple(annotations.shape)}, expected [{B}, M, K] with K >= {ANN_COLS}")
    if annotations.shape[1] > MAX_ROWS:
        raise ValueError(f"retina loss: {annotations.shape[1]} annotation rows per image, at most {MAX_ROWS} supported")
    for t, name in ((cls_scores, "cls_scores"), (reg_preds, "reg_preds"), (anchors, "anchors"), (annotations, "annotations")):
        check(t, "retina loss", name, torch.float32)
    return cls_scores.contiguous(), reg_preds.contiguous(), anchor.contiguous(), annotations.contiguous()


def _forward(cls_scores, reg_preds, anchor, ann, cfg: LossConfig, params: np.ndarray):
    B, N, C = cls_scores.shape
    M, K = ann.shape[1], ann.shape[2]
    dev = cls_scores.device
    ws, ws_bytes = workspace("vd3d_retina_loss_workspace_bytes", B, N, M, device=dev)
    assign = torch.empty(B, N, dtype=torch.int32, device=dev)
    counts = torch.empty(B, 3, dtype=torch.int32, device=dev)
    scale = torch.empty(1, dtype=torch.float32, device=dev)
    cls_loss = torch.empty((), dtype=torch.float32, device=dev)
    reg_loss = torch.empty((), dtype=torch.float32, device=dev)
    _lib.call("vd3d_retina_loss_forward", cls_scores.data_ptr(), reg_preds.data_ptr(), anchor.data_ptr(), ann.data_ptr(), B, N, C, M, K,
              params.ctypes.data, int(cfg.match_low_quality), int(cfg.gt_max_assign_all), ws.data_ptr(), ws_bytes, assign.data_ptr(),
              counts.data_ptr(), scale.data_ptr(), cls_loss.data_ptr(), reg_loss.data_ptr(), stream(cls_scores))
    return cls_loss, reg_loss, assign, counts, scale


class RetinaHeadLoss(torch.autograd.Function):
    """(cls_scores [B,N,C], reg_preds [B,N,4], anchor [N,4], annotations [B,M,K], cfg) -> (cls_loss, reg_loss), both 0-d."""

    @staticmethod
    def forward(ctx, cls_scores, reg_preds, anchor, ann, cfg: LossConfig):
        params = cfg.params()
        cls_loss, reg_loss, assign, _, scale = _forward(cls_scores, reg_preds, anchor, ann, cfg, params)
        ctx.save_for_backward(cls_scores, reg_preds, anchor, ann, assign, scale)
        ctx.params = params
        return cls_loss, reg_loss

    @staticmethod
    def backward(ctx, g_cls, g_reg):
        cls_scores, reg_preds, anchor, ann, assign, scale = ctx.saved_tensors
        grad_out = grad_out_pair(g_cls, g_reg, cls_scores.device)
        B, N, C = cls_scores.shape
        grad_cls = torch.empty_like(cls_scores)
        grad_reg = torch.empty_like(reg_preds)
        _lib.call("vd3d_retina_loss_backward", cls_scores.data_ptr(), reg_preds.data_ptr(), anchor.data_ptr(), ann.data_ptr(), B, N, C,
                  ann.shape[1], ann.shape[2], ctx.params.ctypes.data, assign.data_ptr(), scale.data_ptr(), grad_out.data_ptr(),
                  grad_cls.data_ptr(), grad_reg.data_ptr(), stream(cls_scores))
        return grad_cls, grad_reg, None, None, None


def retinanet_head_loss(cls_scores: torch.Tensor, reg_preds: torch.Tensor, anchors: torch.Tensor, annotations: torch.Tensor, cfg):
    """The reference head's `loss` (retinanet_head.py:309-362).  cls_scores [B,N,C] logits, reg_preds [B,N,4] deltas, anchors:
    `get_anchor`'s [1,N,4] (or [N,4]); annotations [B,M,K], K >= 5 (x1 y1 x2 y2 class first, class -1 = padding; the trainer passes
    compound_annotation's 12 columns); cfg: a LossConfig, or the head's loss_cfg mapping (num_classes = cls_scores' last dimension, default
    target_means / target_stds).  Returns (cls_loss, reg_loss, dict(cls_loss, reg_loss, total_loss)), 0-d float32 tensors differentiable
    in cls_scores and reg_preds."""
    cfg = as_config(LossConfig, cfg, cls_scores.shape[-1])
    cls_scores, reg_preds, anchor, ann = _inputs(cls_scores, reg_preds, anchors, annotations, cfg)
    cls_loss, reg_loss = RetinaHeadLoss.apply(cls_scores, reg_preds, anchor, ann, cfg)
    return cls_loss, reg_loss, dict(cls_loss=cls_loss, reg_loss=reg_loss, total_loss=cls_loss + reg_loss)


def assignment(cls_scores, reg_preds, anchors, annotations, cfg):
    """The forward's anchor assignment and counts (same arguments as retinanet_head_loss): assigned_gt_inds [B, N] int32 (1-based among
    the image's valid annotation rows, 0 negative -- every anchor of an image without a valid row --, -1 ignored) and counts [B, 3] int32
    (positives, negatives, ignored)."""
    cfg = as_config(LossConfig, cfg, cls_scores.shape[-1])
    with torch.no_grad():
        _, _, assign, counts, _ = _forward(*_inputs(cls_scores, reg_preds, anchors, annotations, cfg), cfg, cfg.params())
    return assign, counts


def _head_config(head) -> LossConfig:
    """LossConfig.from_head, cached on the head: reading the balance-weight buffer is a device-to-host copy, so it is redone only when the
    buffer is replaced or written in place (its storage or version counter changes) or a setting changes."""
    bw = head.loss_cls.balance_weights
    key = (bw.data_ptr(), bw._version, head.num_clasess, head.loss_cls.gamma, id(head.loss_cfg), tuple(head.target_means),
           tuple(head.target_stds))
    return cached_on(head, "_vd3d_retina_loss_config", key, lambda: LossConfig.from_head(head))


def head_loss(self, cls_scores, reg_preds, anchors, annotations):
    """Drop-in `RetinanetHead.loss(self, cls_scores, reg_preds, anchors, annotations)` over the native loss."""
    return retinanet_head_loss(cls_scores, reg_preds, anchors, annotations, _head_config(self))
