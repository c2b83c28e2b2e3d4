"""Stereo3D's disparity loss on the GPU: the reference's `DisparityLoss(max_disp)` (R/networks/heads/losses.py:122-135, with
StereoFocalLoss and LaplaceDisp2Prob from R/networks/lib/disparity_loss/*.py; R/ = visualDet3D in the reference tree) as one autograd
Function over csrc/disparity_loss.cu.

The stereo focal loss with a Laplace target (variance 0.5) over the cost volume `depth_output` [B, max_disp, H, W]: the forward reads the
volume once in two launches and keeps each pixel's log-sum-exp; the backward reads it once more and writes the gradient once.  Nothing
synchronises the host (the reference does three times per call: `mask.sum() < 1` and its NaN guard) and no sum uses float atomics, so two
runs give the same bits and the pair can be captured in a CUDA graph.  There is no CPU path.

Only the settings the detector ships are supported, and anything else is refused before a launch: one cost volume (no multi-level list),
start_disp 0, dilation 1, focal_coefficient 0, unit level weights, and a label at the volume's B, H, W (the reference's rescale branch
cannot broadcast against a volume of max_disp channels anyway).  Where the reference raises on a non-finite label, the loss is NaN.

    disparity_loss(est_cost, gt_disp, max_disp=96)  -> 0-dim float32 loss
    forward                                          the method `plugin.install_disparity_loss_into_reference()` binds
"""
from __future__ import annotations

import torch

from . import _lib
from .loss_common import check, stream, workspace

MAX_DISP_LIMIT = 1024       # csrc/disparity_loss.cu keeps a table of D + 1 floats per block


def _is_one(v) -> bool:
    """The reference's `weights` / `dilation` after its first call become one-element lists ([1.0], [1]); both forms mean one level."""
    if isinstance(v, (list, tuple)):
        return len(v) == 1 and _is_one(v[0])
    return v == 1


def check_criterion(criterion) -> None:
    """Refuse StereoFocalLoss settings other than the shipped ones (DisparityLoss builds StereoFocalLoss(max_disp) with the defaults)."""
    if criterion.focal_coefficient != 0:
        raise ValueError(f"disparity loss: focal_coefficient {criterion.focal_coefficient} is not supported (the shipped value is 0)")
    if criterion.start_disp != 0:
        raise ValueError(f"disparity loss: start_disp {criterion.start_disp} is not supported (the shipped value is 0)")
    if not _is_one(criterion.dilation):
        raise ValueError(f"disparity loss: dilation {criterion.dilation} is not supported (the shipped value is 1)")
    if not (criterion.weights is None or _is_one(criterion.weights)):
        raise ValueError(f"disparity loss: level weights {criterion.weights} are not supported (one level of weight 1)")


def _inputs(est_cost, gt_disp, max_disp):
    """Validated (cost, label [B, H, W]); raises before any launch."""
    if isinstance(est_cost, (list, tuple)):
        raise ValueError("disparity loss: a list of cost volumes (multi-level) is not supported; pass one [B, max_disp, H, W] tensor")
    if not isinstance(est_cost, torch.Tensor) or not isinstance(gt_disp, torch.Tensor):
        raise TypeError("disparity loss: est_cost and gt_disp must be tensors")
    if not isinstance(max_disp, int) or not 2 <= max_disp <= MAX_DISP_LIMIT:
        raise ValueError(f"disparity loss: max_disp must be an int in [2, {MAX_DISP_LIMIT}], got {max_disp!r}")
    if est_cost.dim() != 4:
        raise ValueError(f"disparity loss: est_cost must be [B, max_disp, H, W], got {tuple(est_cost.shape)}")
    B, D, H, W = est_cost.shape
    if D != max_disp:
        raise ValueError(f"disparity loss: est_cost has {D} channels, max_disp is {max_disp} (the reference cannot broadcast them)")
    label = gt_disp
    if label.dim() == 4 and label.shape[1] == 1:
        label = label[:, 0]
    if tuple(label.shape) != (B, H, W):
        raise ValueError(f"disparity loss: gt_disp {tuple(gt_disp.shape)} does not match est_cost's B, H, W = {(B, H, W)} (no rescaled "
                         "label is supported)")
    for name, t in (("est_cost", est_cost), ("gt_disp", gt_disp)):             # both dtypes before either device
        if t.dtype != torch.float32:
            raise RuntimeError(f"disparity loss: {name} must be float32, got {t.dtype}")
    for name, t in (("est_cost", est_cost), ("gt_disp", gt_disp)):
        check(t, "disparity loss", name, torch.float32)
    if est_cost.device != gt_disp.device:
        raise RuntimeError(f"disparity loss: est_cost on {est_cost.device}, gt_disp on {gt_disp.device}")
    return est_cost, label


class DisparityLossFn(torch.autograd.Function):
    """(cost [B, D, H, W], label [B, H, W]) -> 0-dim loss; differentiable in cost."""

    @staticmethod
    def forward(ctx, cost, label):
        cost, label = cost.contiguous(), label.contiguous()
        B, D, H, W = cost.shape
        ws, ws_bytes = workspace("vd3d_disparity_loss_workspace_bytes", B, D, H, W, device=cost.device)
        lse = torch.empty((B, H, W), dtype=torch.float32, device=cost.device)
        loss = torch.empty((), dtype=torch.float32, device=cost.device)
        _lib.call("vd3d_disparity_loss_forward", cost.data_ptr(), label.data_ptr(), B, D, H, W, ws.data_ptr(), ws_bytes, lse.data_ptr(),
                  loss.data_ptr(), stream(cost))
        ctx.save_for_backward(cost, label, lse)
        return loss

    @staticmethod
    def backward(ctx, g):
        cost, label, lse = ctx.saved_tensors
        B, D, H, W = cost.shape
        g = g.float().contiguous()
        grad = torch.empty_like(cost)
        _lib.call("vd3d_disparity_loss_backward", cost.data_ptr(), label.data_ptr(), lse.data_ptr(), B, D, H, W, g.data_ptr(),
                  grad.data_ptr(), stream(cost))
        return grad, None


def disparity_loss(est_cost: torch.Tensor, gt_disp: torch.Tensor, max_disp: int = 96) -> torch.Tensor:
    """`DisparityLoss(max_disp)(est_cost, gt_disp)` of the reference.  est_cost: [B, max_disp, H, W] float32 CUDA logits (not
    normalised); gt_disp: [B, H, W] or [B, 1, H, W] float32 disparity at the same H, W (0 = no label).  Returns the 0-dim float32 loss,
    differentiable in est_cost; 0 when no pixel has 0 < gt_disp < max_disp, NaN when a label value is not finite."""
    cost, label = _inputs(est_cost, gt_disp, max_disp)
    return DisparityLossFn.apply(cost, label)


def forward(self, x, label):
    """Drop-in `DisparityLoss.forward(self, x, label)`: moves the label to the GPU like the reference, and reads the criterion's max_disp
    and settings."""
    check_criterion(self.criterion)
    label = label.cuda()
    return disparity_loss(x, label, self.criterion.max_disp)
