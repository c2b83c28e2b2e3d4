"""Training loss of the KM3D head on the GPU: the reference's `KM3DHead.loss` (R/networks/heads/km3d_head.py:316-351, with Position_loss
and gen_position from R/networks/utils/rtm3d_utils.py:230-455; R/ = visualDet3D in the reference tree) as one autograd Function over
csrc/km3d_loss.cu.

The two heatmap focal losses (hm, hm_hp), the weighted-L1 keypoint loss, the L1 losses (wh, dim, reg, hp_offset), the rotation bin /
residual loss and the position terms (the least-squares position of each row against its location, the 3-D IoU of each row's own box
pair, the probability loss against that IoU) run in three launches with no host synchronisation; the backward is one launch that writes
all nine gradient maps, the position loss's included (through the least-squares solve).  The maps are read at `ind` / `hp_ind` in their
NCHW layout.  Sums are reduced in a fixed order without float atomics, so two runs give the same bits and the pair can be captured in a
CUDA graph (the graph then holds one epoch's exp_rampup weight).  There is no CPU path.

Differences from the reference: the annotations are not modified (the reference rewrites annotations['dep'] in place through
_RegWeightedL1Loss); the least-squares solve adds no jitter (the reference adds randn * 1e-8 to A^T A); the box score is the IoU of each
row's own pair instead of the diagonal of a (B*K) x (B*K) IoU matrix.

    km3d_head_loss(output, annotations, P2, epoch, cfg)  -> (loss 0-dim, loss_stats: the reference's 13 keys, 0-dim f32)
    head_loss                                            the method `plugin.install_km3d_loss_into_reference()` binds
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Mapping

import numpy as np
import torch

from . import _lib
from .loss_common import as_config, map_inputs, ptr_array, stream, workspace

MAPS = (("hm", None), ("wh", 2), ("hps", 18), ("rot", 8), ("dim", 3), ("prob", 1), ("reg", 2), ("hm_hp", 9), ("hp_offset", 2))
TERMS = ("hm_loss", "hp_loss", "hm_hp_loss", "hp_offset_loss", "wh_loss", "off_loss", "dim_loss", "rot_loss", "prob_loss", "coor_loss",
         "box_score")
MAX_ROWS = 128
NUM_JOINTS = 9
_HM_TARGETS = (("hm", None), ("hm_hp", NUM_JOINTS))        # [B, channels (None: C), H, W] like the output
# annotation key -> (dtypes accepted, trailing shape after [B, rows], rows per object: 1 or 9)
_TARGETS = (("ind", (torch.int64,), (), 1), ("reg_mask", (torch.uint8, torch.bool), (), 1), ("hps", (torch.float32,), (18,), 1),
            ("hps_mask", (torch.uint8, torch.bool), (18,), 1), ("dep", (torch.float32,), (1,), 1), ("rotbin", (torch.int64,), (2,), 1),
            ("rotres", (torch.float32,), (2,), 1), ("wh", (torch.float32,), (2,), 1), ("dim", (torch.float32,), (3,), 1),
            ("reg", (torch.float32,), (2,), 1), ("hp_ind", (torch.int64,), (), NUM_JOINTS),
            ("hp_mask", (torch.uint8, torch.bool), (), NUM_JOINTS), ("hp_offset", (torch.float32,), (2,), NUM_JOINTS),
            ("location", (torch.float32,), (3,), 1), ("ori", (torch.float32,), (1,), 1))


@dataclass(frozen=True)
class LossConfig:
    """The settings the reference's loss reads: `build_loss(gamma=2.0, output_w=1280, rampup_length=100)` (km3d_head.py:44-51)."""
    output_w: float = 1280.0
    rampup_length: float = 100.0

    def __post_init__(self):
        if not self.output_w > 0:
            raise ValueError(f"km3d loss: output_w must be > 0, got {self.output_w}")
        if not self.rampup_length >= 0:
            raise ValueError(f"km3d loss: rampup_length must be >= 0, got {self.rampup_length}")

    @classmethod
    def from_loss_cfg(cls, loss_cfg: Mapping) -> "LossConfig":
        """From a config's `head.loss_cfg` (R/config/KM3D_example: head_loss)."""
        return cls(output_w=float(loss_cfg.get("output_w", 1280)), rampup_length=float(loss_cfg.get("rampup_length", 100)))

    @classmethod
    def from_head(cls, head) -> "LossConfig":
        """From a reference KM3DHead's own attributes (what its `loss` reads)."""
        return cls(output_w=float(head.position_loss.output_w), rampup_length=float(head.rampup_length))

    def exp_rampup(self, epoch) -> float:
        """KM3DHead.exp_rampup (km3d_head.py:53-59), on the host: the weight of prob_loss and coor_loss."""
        if epoch < self.rampup_length:
            epoch = np.clip(epoch, 0.0, self.rampup_length)
            phase = 1.0 - epoch / self.rampup_length
            return float(np.exp(-5.0 * phase * phase))
        return 1.0


class KM3DLoss(torch.autograd.Function):
    """(output_w, rampup, targets tuple, sizes, *maps) -> (total 0-dim, terms [11]); differentiable in the nine maps."""

    @staticmethod
    def forward(ctx, output_w: float, rampup: float, targets, sizes, *maps):
        dev = maps[0].device
        ws, ws_bytes = workspace("vd3d_km3d_loss_workspace_bytes", *sizes, device=dev)
        terms = torch.empty(len(TERMS), dtype=torch.float32, device=dev)
        total = torch.empty((), dtype=torch.float32, device=dev)
        _lib.call("vd3d_km3d_loss_forward", ptr_array(maps), ptr_array(targets), *sizes, output_w, rampup, ws.data_ptr(), ws_bytes,
                  terms.data_ptr(), total.data_ptr(), stream(maps[0]))
        ctx.save_for_backward(ws, *targets, *maps)
        ctx.args, ctx.sizes, ctx.n_targets = (output_w, rampup), sizes, len(targets)
        ctx.set_materialize_grads(False)
        return total, terms

    @staticmethod
    def backward(ctx, g_total, g_terms):
        ws, *rest = ctx.saved_tensors
        targets, maps = rest[:ctx.n_targets], rest[ctx.n_targets:]
        grads = [torch.empty_like(m) for m in maps]
        g_total = None if g_total is None else g_total.float().contiguous()
        g_terms = None if g_terms is None else g_terms.float().contiguous()
        _lib.call("vd3d_km3d_loss_backward", ptr_array(maps), ptr_array(targets), *ctx.sizes, *ctx.args, ws.data_ptr(),
                  None if g_terms is None else g_terms.data_ptr(), None if g_total is None else g_total.data_ptr(), ptr_array(grads),
                  stream(maps[0]))
        return (None, None, None, None, *grads)


def km3d_head_loss(output: Mapping, annotations: Mapping, P2: torch.Tensor, epoch=0, cfg=None):
    """The reference head's `loss` (km3d_head.py:316-351).  output: the head's nine maps (fp32 NCHW, hm / hm_hp as logits); annotations:
    the KittiRTM3DDataset targets (ind / hp_ind / rotbin int64, masks uint8 or bool); P2 [B, 3, 4]; epoch: what exp_rampup reads; cfg: a
    LossConfig or the head's loss_cfg mapping (None: the defaults).  Returns (loss, loss_stats) like the reference: 0-dim float32 device
    tensors, loss_stats with `loss` (= box_score), the ten unweighted terms, box_score and total_loss (= loss); box_score carries no
    gradient.  The annotations are not modified."""
    cfg = as_config(LossConfig, cfg or {})
    maps, targets, sizes = map_inputs("km3d loss", "KM3D", MAPS, _HM_TARGETS, _TARGETS, MAX_ROWS, output, annotations, P2)
    total, terms = KM3DLoss.apply(float(cfg.output_w), cfg.exp_rampup(epoch), tuple(targets), sizes, *maps)
    stats = {name: terms[i] for i, name in enumerate(TERMS)}
    stats = dict(loss=stats["box_score"], **stats)
    stats["total_loss"] = total
    return total, stats


def head_loss(self, output, annotations, meta):
    """Drop-in `KM3DHead.loss(self, output, annotations, meta)` over the native loss: reads meta['P2'] and meta['epoch'] and the head's
    position_loss.output_w and rampup_length."""
    return km3d_head_loss(output, annotations, meta["P2"], meta["epoch"], LossConfig.from_head(self))
