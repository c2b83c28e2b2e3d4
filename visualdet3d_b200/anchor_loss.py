"""Training loss of the 3-D anchor head on the GPU: the reference's `AnchorBasedDetection3DHead.loss`
(R/networks/heads/detection_3d_head.py:402-498; R/ = visualDet3D in the reference tree), which StereoHead (Stereo3D) and
GroundAwareHead (Yolo3D, GroundAwareYolo3D) inherit, as one autograd Function over csrc/anchor_loss.cu.

The anchor assignment (calc_iou, _assign with low-quality matching), the prior's z_mean > 0 selection, _encode, the sigmoid focal,
modified smooth-L1 and alpha BCE terms and the batch reduction run in four launches with no host synchronisation; the backward is one
launch.  Sums are reduced in a fixed order without float atomics, so two runs give the same bits and the pair can be captured in a
CUDA graph.  There is no CPU path.

    anchor3d_head_loss(cls_scores, reg_preds, anchors, annotations, loss_cfg)  -> (cls_loss [1], reg_loss [1], loss dict)
    assignment(...)                                                            -> (assigned_gt_inds [B, N] i32, counts [B, 3] i32)
    head_loss                                                                  the method `plugin.install_loss_into_reference()` binds
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Mapping, Tuple

import numpy as np
import torch

from . import _lib
from .loss_common import as_config, cached_on, check, grad_out_pair, stream, workspace

N_REG = 12          # regression outputs per anchor
N_TERMS = 13        # the 12 smooth-L1 terms and the alpha BCE: the length regression_weight must have
MAX_CLASSES = 8


@dataclass(frozen=True)
class LossConfig:
    """The settings the reference's loss reads, with `_assign` / `build_loss` defaults (detection_3d_head.py:90-107)."""
    num_classes: int
    fg_iou_threshold: float = 0.5
    bg_iou_threshold: float = 0.0
    min_iou_threshold: float = 0.0
    match_low_quality: bool = True
    gt_max_assign_all: bool = True
    focal_loss_gamma: float = 0.0
    balance_weights: Tuple[float, ...] = (0.0,)
    regression_weight: Tuple[float, ...] = (1.0,) * N_TERMS
    l1_regression_alpha: float = 9.0

    def __post_init__(self):
        if not 1 <= self.num_classes <= MAX_CLASSES:
            raise ValueError(f"anchor loss: num_classes must be in 1..{MAX_CLASSES}, got {self.num_classes}")
        if len(self.balance_weights) not in (1, self.num_classes):
            raise ValueError(f"anchor loss: balance_weight has {len(self.balance_weights)} entries; it needs 1 or num_classes "
                             f"({self.num_classes})")
        if len(self.regression_weight) != N_TERMS:
            raise ValueError(f"anchor loss: regression_weight has {len(self.regression_weight)} entries; the loss has {N_TERMS} terms "
                             "(12 regression outputs and the alpha classification)")

    @classmethod
    def from_loss_cfg(cls, loss_cfg: Mapping, num_classes: int) -> "LossConfig":
        """From a config's `head.loss_cfg` (R/config/*_example: head_loss)."""
        get = loss_cfg.get
        if get("decode_before_loss", False):
            raise ValueError("anchor loss: loss_cfg.decode_before_loss=True is not supported (the reference's branch indexes the "
                             "unmasked anchor table with masked indices, detection_3d_head.py:466-471)")
        return cls(num_classes=int(num_classes),
                   fg_iou_threshold=float(get("fg_iou_threshold", 0.5)),
                   bg_iou_threshold=float(get("bg_iou_threshold", 0.0)),
                   min_iou_threshold=float(get("min_iou_threshold", 0.0)),
                   match_low_quality=bool(get("match_low_quality", True)),
                   gt_max_assign_all=bool(get("gt_max_assign_all", True)),
                   focal_loss_gamma=float(get("focal_loss_gamma", 0.0)),
                   balance_weights=tuple(float(v) for v in get("balance_weight", [0])),
                   regression_weight=tuple(float(v) for v in get("regression_weight", [1.0] * N_TERMS)),
                   l1_regression_alpha=float(get("L1_regression_alpha", 9)))

    @classmethod
    def from_head(cls, head) -> "LossConfig":
        """From a reference head's own attributes (what its `loss` reads): num_classes, loss_cfg, focal_loss_gamma, the balance_weights /
        regression_weight buffers and loss_bbox.alpha."""
        if getattr(head, "decode_before_loss", False):
            raise ValueError("anchor loss: loss_cfg.decode_before_loss=True is not supported (the reference's branch indexes the "
                             "unmasked anchor table with masked indices, detection_3d_head.py:466-471)")
        lc = head.loss_cfg
        return cls(num_classes=int(head.num_classes),
                   fg_iou_threshold=float(lc.get("fg_iou_threshold", 0.5)),
                   bg_iou_threshold=float(lc.get("bg_iou_threshold", 0.0)),
                   min_iou_threshold=float(lc.get("min_iou_threshold", 0.0)),
                   match_low_quality=bool(lc.get("match_low_quality", True)),
                   gt_max_assign_all=bool(lc.get("gt_max_assign_all", True)),
                   focal_loss_gamma=float(head.focal_loss_gamma),
                   balance_weights=tuple(float(v) for v in head.balance_weights.reshape(-1).tolist()),
                   regression_weight=tuple(float(v) for v in head.regression_weight.reshape(-1).tolist()),
                   l1_regression_alpha=float(head.loss_bbox.alpha))

    def params(self) -> np.ndarray:
        """The float32 parameter block of vd3d_anchor_loss_forward / _backward (include/vd3d_b200.h)."""
        a = self.l1_regression_alpha
        bw = self.balance_weights * (self.num_classes if len(self.balance_weights) == 1 else 1)
        return np.ascontiguousarray(np.array([self.fg_iou_threshold, self.bg_iou_threshold, self.min_iou_threshold, self.focal_loss_gamma,
                                              1.0 / a, 0.5 * a, 0.5 / a, *bw, *self.regression_weight], dtype=np.float32))


def _inputs(cls_scores, reg_preds, anchors: Mapping, annotations, cfg: LossConfig):
    check(cls_scores, "anchor loss", "cls_scores", torch.float32)
    check(reg_preds, "anchor loss", "reg_preds", torch.float32)
    anchor = anchors["anchors"][0].contiguous()
    mask = anchors["mask"].contiguous()
    mean_std = anchors["anchor_mean_std_3d"].contiguous()
    ann = annotations.contiguous()
    check(anchor, "anchor loss", "anchors['anchors']", torch.float32)
    check(mask, "anchor loss", "anchors['mask']", torch.bool)
    check(mean_std, "anchor loss", "anchors['anchor_mean_std_3d']", torch.float32)
    check(ann, "anchor loss", "annotations", torch.float32)
    B, N, C1 = cls_scores.shape
    C = cfg.num_classes
    if C1 != C + 1:
        raise ValueError(f"anchor loss: cls_scores has {C1} columns, expected num_classes + 1 = {C + 1}")
    if tuple(reg_preds.shape) != (B, N, N_REG):
        raise ValueError(f"anchor loss: reg_preds {tuple(reg_preds.shape)}, expected {(B, N, N_REG)}")
    if tuple(anchor.shape) != (N, 4) or tuple(mask.shape) != (B, N) or tuple(mean_std.shape) != (N, C, 6, 2):
        raise ValueError(f"anchor loss: anchors {tuple(anchor.shape)} / mask {tuple(mask.shape)} / anchor_mean_std_3d "
                         f"{tuple(mean_std.shape)} do not match {B} images x {N} anchors x {C} classes")
    if ann.dim() != 3 or ann.shape[0] != B or ann.shape[2] != 12:
        raise ValueError(f"anchor loss: annotations {tuple(ann.shape)}, expected [{B}, M, 12]")
    return cls_scores.contiguous(), reg_preds.contiguous(), anchor, mask, mean_std, ann


def _forward(cls_scores, reg_preds, anchor, mask, mean_std, ann, cfg: LossConfig, params: np.ndarray):
    B, N, _ = cls_scores.shape
    M = ann.shape[1]
    dev = cls_scores.device
    ws, ws_bytes = workspace("vd3d_anchor_loss_workspace_bytes", B, N, M, device=dev)
    assign = torch.empty(B, N, dtype=torch.int32, device=dev)
    counts = torch.empty(B, 3, dtype=torch.int32, device=dev)
    factors = torch.empty(B, 2, dtype=torch.float32, device=dev)
    cls_loss = torch.empty(1, dtype=torch.float32, device=dev)
    reg_loss = torch.empty(1, dtype=torch.float32, device=dev)
    _lib.call("vd3d_anchor_loss_forward", cls_scores.data_ptr(), reg_preds.data_ptr(), anchor.data_ptr(), mask.data_ptr(),
              mean_std.data_ptr(), ann.data_ptr(), B, N, cfg.num_classes, M, params.ctypes.data, int(cfg.match_low_quality),
              int(cfg.gt_max_assign_all), ws.data_ptr(), ws_bytes, assign.data_ptr(), counts.data_ptr(), factors.data_ptr(),
              cls_loss.data_ptr(), reg_loss.data_ptr(), stream(cls_scores))
    return cls_loss, reg_loss, assign, counts, factors


class AnchorHeadLoss(torch.autograd.Function):
    """(cls_scores, reg_preds, anchor [N,4], mask [B,N], mean_std, annotations, cfg) -> (cls_loss [1], reg_loss [1])."""

    @staticmethod
    def forward(ctx, cls_scores, reg_preds, anchor, mask, mean_std, ann, cfg: LossConfig):
        params = cfg.params()
        cls_loss, reg_loss, assign, _, factors = _forward(cls_scores, reg_preds, anchor, mask, mean_std, ann, cfg, params)
        ctx.save_for_backward(cls_scores, reg_preds, anchor, mean_std, ann, assign, factors)
        ctx.cfg, ctx.params = cfg, params
        return cls_loss, reg_loss

    @staticmethod
    def backward(ctx, g_cls, g_reg):
        cls_scores, reg_preds, anchor, mean_std, ann, assign, factors = ctx.saved_tensors
        grad_out = grad_out_pair(g_cls, g_reg, cls_scores.device)
        B, N, C1 = cls_scores.shape
        grad_cls = torch.empty_like(cls_scores)
        grad_reg = torch.empty_like(reg_preds)
        _lib.call("vd3d_anchor_loss_backward", cls_scores.data_ptr(), reg_preds.data_ptr(), anchor.data_ptr(), mean_std.data_ptr(),
                  ann.data_ptr(), B, N, ctx.cfg.num_classes, ann.shape[1], ctx.params.ctypes.data, assign.data_ptr(), factors.data_ptr(),
                  grad_out.data_ptr(), grad_cls.data_ptr(), grad_reg.data_ptr(), stream(cls_scores))
        return grad_cls, grad_reg, None, None, None, None, None


def anchor3d_head_loss(cls_scores: torch.Tensor, reg_preds: torch.Tensor, anchors: Mapping, annotations: torch.Tensor, cfg):
    """The reference head's `loss` (detection_3d_head.py:402-498).  anchors: `get_anchor`'s dict (anchors [1,N,4], mask [B,N],
    anchor_mean_std_3d [N,C,6,2]); annotations [B,M,12] compound_annotation rows (class -1 = padding); cfg: the head's loss_cfg
    mapping (num_classes = cls_scores' last dimension - 1) or a LossConfig.  Returns (cls_loss [1], reg_loss [1],
    dict(cls_loss, reg_loss, total_loss)), differentiable in cls_scores and reg_preds."""
    cfg = as_config(LossConfig, cfg, cls_scores.shape[-1] - 1)
    cls_scores, reg_preds, anchor, mask, mean_std, ann = _inputs(cls_scores, reg_preds, anchors, annotations, cfg)
    cls_loss, reg_loss = AnchorHeadLoss.apply(cls_scores, reg_preds, anchor, mask, mean_std, ann, cfg)
    return cls_loss, reg_loss, dict(cls_loss=cls_loss, reg_loss=reg_loss, total_loss=cls_loss + reg_loss)


def assignment(cls_scores, reg_preds, anchors: Mapping, annotations, cfg):
    """The forward's anchor assignment and counts (same arguments as anchor3d_head_loss): assigned_gt_inds [B, N] int32 (1-based among
    the image's valid annotation rows, 0 negative, -1 ignored or image without ground truth, -2 outside the mask) and counts [B, 3]
    int32 (positives assigned, positives kept by the prior's z_mean > 0 selection, negatives)."""
    cfg = as_config(LossConfig, cfg, cls_scores.shape[-1] - 1)
    with torch.no_grad():
        _, _, assign, counts, _ = _forward(*_inputs(cls_scores, reg_preds, anchors, annotations, cfg), cfg, cfg.params())
    return assign, counts


def _head_config(head) -> LossConfig:
    """LossConfig.from_head, cached on the head: reading the weight buffers is a device-to-host copy, so it is redone only when a buffer
    is replaced or written in place (its storage or version counter changes)."""
    key = tuple((t.data_ptr(), t._version) for t in (head.balance_weights, head.regression_weight)) + (
        head.num_classes, head.focal_loss_gamma, head.decode_before_loss, id(head.loss_cfg), head.loss_bbox.alpha)
    return cached_on(head, "_vd3d_loss_config", key, lambda: LossConfig.from_head(head))


def head_loss(self, cls_scores, reg_preds, anchors, annotations, P2s):
    """Drop-in `AnchorBasedDetection3DHead.loss(self, cls_scores, reg_preds, anchors, annotations, P2s)` over the native loss."""
    return anchor3d_head_loss(cls_scores, reg_preds, anchors, annotations, _head_config(self))
