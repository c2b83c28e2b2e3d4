"""Training loss of the MonoFlex head on the GPU: the reference's `MonoFlexHead.loss` (R/networks/heads/monoflex_head.py:181-236;
R/ = visualDet3D in the reference tree) as one autograd Function over csrc/monoflex_loss.cu.

The heatmap focal loss, the weighted-L1 keypoint loss, the rotation bin / residual loss and the six terms of the rows with reg_mask set
(IoU box, dimension, offset, Laplacian depth, keypoint depth, merged depth) run in three launches with no host synchronisation; the
backward is one launch that writes all nine gradient maps.  The maps are read at `ind` in their NCHW layout.  Sums are reduced in a
fixed order without float atomics, so two runs give the same bits and the pair can be captured in a CUDA graph.  There is no CPU path.

    monoflex_head_loss(output, annotations, P2, cfg)  -> (loss 0-dim, loss_stats: the nine terms and total_loss, 0-dim f32)
    head_loss                                         the method `plugin.install_monoflex_loss_into_reference()` binds
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Mapping, Tuple

import torch

from . import _lib
from .loss_common import as_config, map_inputs, ptr_array, stream, workspace

MAPS = (("hm", None), ("bbox2d", 4), ("hps", 20), ("rot", 8), ("dim", 3), ("reg", 2), ("depth", 1), ("depth_uncertainty", 1),
        ("corner_uncertainty", 3))
TERMS = ("hm_loss", "hp_loss", "box2d_loss", "off_loss", "dim_loss", "depth_loss", "kpd_loss", "rot_loss", "soft_depth_loss")
MAX_ROWS = 128
# annotation key -> (dtypes accepted, trailing shape after [B, K], rows per object); hm is [B, C, H, W] like the output
_TARGETS = (("ind", (torch.int64,), (), 1), ("reg_mask", (torch.bool, torch.uint8), (), 1), ("hps", (torch.float32,), (20,), 1),
            ("hps_mask", (torch.uint8, torch.bool), (20,), 1), ("dep", (torch.float32,), (1,), 1), ("rotbin", (torch.int64,), (2,), 1),
            ("rotres", (torch.float32,), (2,), 1), ("bboxes2d_target", (torch.float32,), (4,), 1), ("dim", (torch.float32,), (3,), 1),
            ("reg", (torch.float32,), (2,), 1), ("kp_detph_mask", (torch.float32,), (3,), 1))


@dataclass(frozen=True)
class LossConfig:
    """The settings the reference's loss reads: `build_loss(uncertainty_range=[-10, 10], uncertainty_weight=1.0)`
    (monoflex_head.py:17-24)."""
    uncertainty_range: Tuple[float, float] = (-10.0, 10.0)
    uncertainty_weight: float = 1.0

    def __post_init__(self):
        if len(self.uncertainty_range) != 2 or not self.uncertainty_range[1] >= self.uncertainty_range[0]:
            raise ValueError(f"monoflex loss: uncertainty_range must be [low, high] with high >= low, got {self.uncertainty_range}")

    @classmethod
    def from_loss_cfg(cls, loss_cfg: Mapping) -> "LossConfig":
        """From a config's `head.loss_cfg` (R/config/Monoflex_example: head_loss)."""
        r = loss_cfg.get("uncertainty_range", (-10.0, 10.0))
        return cls(uncertainty_range=tuple(float(v) for v in r), uncertainty_weight=float(loss_cfg.get("uncertainty_weight", 1.0)))

    @classmethod
    def from_head(cls, head) -> "LossConfig":
        """From a reference MonoFlexHead's own attributes (what its `loss` reads)."""
        return cls(uncertainty_range=tuple(float(v) for v in head.uncertainty_range), uncertainty_weight=float(head.uncertainty_weight))


class MonoFlexLoss(torch.autograd.Function):
    """(cfg, targets tuple, *maps) -> (total 0-dim, terms [9]); differentiable in the nine maps."""

    @staticmethod
    def forward(ctx, cfg: LossConfig, targets, sizes, *maps):
        dev = maps[0].device
        ws, ws_bytes = workspace("vd3d_monoflex_loss_workspace_bytes", *sizes, device=dev)
        terms = torch.empty(len(TERMS), dtype=torch.float32, device=dev)
        total = torch.empty((), dtype=torch.float32, device=dev)
        lo, hi = cfg.uncertainty_range
        _lib.call("vd3d_monoflex_loss_forward", ptr_array(maps), ptr_array(targets), *sizes, lo, hi, cfg.uncertainty_weight,
                  ws.data_ptr(), ws_bytes, terms.data_ptr(), total.data_ptr(), stream(maps[0]))
        ctx.save_for_backward(ws, *targets, *maps)
        ctx.cfg, ctx.sizes, ctx.n_targets = cfg, sizes, len(targets)
        ctx.set_materialize_grads(False)
        return total, terms

    @staticmethod
    def backward(ctx, g_total, g_terms):
        ws, *rest = ctx.saved_tensors
        targets, maps = rest[:ctx.n_targets], rest[ctx.n_targets:]
        grads = [torch.empty_like(m) for m in maps]
        g_total = None if g_total is None else g_total.float().contiguous()
        g_terms = None if g_terms is None else g_terms.float().contiguous()
        lo, hi = ctx.cfg.uncertainty_range
        _lib.call("vd3d_monoflex_loss_backward", ptr_array(maps), ptr_array(targets), *ctx.sizes, lo, hi, ctx.cfg.uncertainty_weight,
                  ws.data_ptr(), None if g_terms is None else g_terms.data_ptr(), None if g_total is None else g_total.data_ptr(),
                  ptr_array(grads), stream(maps[0]))
        return (None, None, None, *grads)


def monoflex_head_loss(output: Mapping, annotations: Mapping, P2: torch.Tensor, cfg=None):
    """The reference head's `loss` (monoflex_head.py:181-236).  output: the head's nine maps (fp32 NCHW, hm as logits); annotations:
    the KittiMonoFlexDataset targets with `ind` int64 and `reg_mask` bool / uint8; P2 [B, 3, 4]; cfg: a LossConfig or the head's
    loss_cfg mapping (None: the defaults).  Returns (loss, loss_stats) like the reference: 0-dim float32 device tensors, loss_stats with
    the nine unweighted terms and total_loss (= loss), all differentiable in the nine maps."""
    cfg = as_config(LossConfig, cfg or {})
    maps, targets, sizes = map_inputs("monoflex loss", "MonoFlex", MAPS, (("hm", None),), _TARGETS, MAX_ROWS, output, annotations, P2)
    total, terms = MonoFlexLoss.apply(cfg, tuple(targets), sizes, *maps)
    stats = {name: terms[i] for i, name in enumerate(TERMS)}
    stats["total_loss"] = total
    return total, stats


def head_loss(self, output, annotations, meta):
    """Drop-in `MonoFlexHead.loss(self, output, annotations, meta)` over the native loss.  Like the reference it rewrites
    annotations['ind'] to int64 and annotations['reg_mask'] to bool; meta['epoch'] is not used by MonoFlex's loss."""
    annotations["ind"] = annotations["ind"].long()
    annotations["reg_mask"] = annotations["reg_mask"].bool()
    return monoflex_head_loss(output, annotations, meta["P2"], LossConfig.from_head(self))
