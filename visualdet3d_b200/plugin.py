"""Plugin surface of the B200 path: the six named registries the reference's scripts look detectors up in.

Contract mirrored from R/visualDet3D/networks/utils/registry.py:21-50 (behaviour, not code):
  * objects are keyed by their ``__name__``; only classes and plain functions are accepted (TypeError otherwise);
  * registering a taken name raises KeyError unless ``force=True``;
  * ``registry[name]`` raises KeyError for unknown names, ``registry.get(name)`` returns None;
  * ``@registry.register_module`` is a bare decorator returning the object unchanged.
Detectors are then built exactly like the reference does: ``DETECTOR_DICT[cfg.detector.name](cfg.detector)``
(R/scripts/train.py:87, R/scripts/eval.py:37).
"""
from __future__ import annotations

import inspect
from typing import Any, Callable, Dict, Iterator, Optional


class Registry:
    __slots__ = ("_name", "_items")

    def __init__(self, name: str):
        self._name = name
        self._items: Dict[str, Any] = {}

    # -- introspection -----------------------------------------------------------------------------------
    @property
    def name(self) -> str:
        return self._name

    @property
    def module_dict(self) -> Dict[str, Any]:
        return self._items

    def __repr__(self) -> str:
        return f"Registry(name={self._name}, items={list(self._items)})"

    def __iter__(self) -> Iterator[str]:
        return iter(self._items)

    def __len__(self) -> int:
        return len(self._items)

    def __contains__(self, key: str) -> bool:
        return key in self._items

    # -- lookup --------------------------------------------------------------------------------------------
    def __getitem__(self, key: str) -> Any:
        return self._items[key]          # KeyError for unknown names, like the reference

    def get(self, key: str) -> Optional[Any]:
        return self._items.get(key)

    # -- registration ----------------------------------------------------------------------------------------
    def _register_module(self, obj: Any, force: bool = False) -> None:
        if not (inspect.isclass(obj) or inspect.isfunction(obj)):
            raise TypeError(f"module must be a class or function, but got {type(obj)}")
        key = obj.__name__
        if key in self._items and not force:
            raise KeyError(f"{key} is already registered in {self._name}")
        self._items[key] = obj

    def register_module(self, obj: Callable = None):
        self._register_module(obj)
        return obj


DATASET_DICT, BACKBONE_DICT, DETECTOR_DICT = Registry("datasets"), Registry("backbones"), Registry("detectors")
PIPELINE_DICT, AUGMENTATION_DICT, SAMPLER_DICT = Registry("pipelines"), Registry("augmentation"), Registry("sampler")


# detectors that replace the reference's class only on request (install_retinanet_into_reference)
OPT_IN_DETECTORS = ("RetinaNet",)


def install_into_reference(force: bool = True):
    """Put every B200 3-D detector / pipeline into the REFERENCE's registries (when `visualDet3D` is importable) so the
    reference's own scripts/eval.py and scripts/train.py pick them up by `cfg.detector.name` with no edit.  The 2-D RetinaNet is
    opt-in: `install_retinanet_into_reference()`."""
    from visualDet3D.networks.utils import registry as ref   # ImportError if the reference is not on sys.path
    for name, cls in DETECTOR_DICT.module_dict.items():
        if name not in OPT_IN_DETECTORS:
            ref.DETECTOR_DICT._register_module(cls, force=force)
    for fn in PIPELINE_DICT.module_dict.values():
        ref.PIPELINE_DICT._register_module(fn, force=force)
    return ref


def install_evaluator_into_reference():
    """Make the REFERENCE's KITTI evaluation run on the native evaluator (`kitti_eval.evaluate`, same signature and strings):
    rebinds `visualDet3D.evaluator.kitti.evaluate.evaluate` and the name `evaluators.py` imported from it at module level, so the
    unmodified `evaluate_kitti_obj` (scripts/eval.py, and scripts/train.py after each evaluation epoch) uses it."""
    from visualDet3D.evaluator.kitti import evaluate as ref_evaluate      # ImportError if the reference is not on sys.path
    from visualDet3D.networks.pipelines import evaluators as ref_evaluators
    from .kitti_eval import evaluate
    ref_evaluate.evaluate = evaluate
    ref_evaluators.evaluate = evaluate
    return evaluate


def install_retinanet_into_reference():
    """Make the REFERENCE's `DETECTOR_DICT['RetinaNet']` the native 2-D RetinaNet, so the unmodified scripts/eval.py (test_mono_detection,
    test_one's 2-D branch) run the RetinaNet config on the GPU path.  Returns the installed class."""
    from visualDet3D.networks.utils import registry as ref   # ImportError if the reference is not on sys.path
    from .detectors.retinanet import RetinaNet
    ref.DETECTOR_DICT._register_module(RetinaNet, force=True)
    return RetinaNet


def install_loss_into_reference():
    """Make the REFERENCE's 3-D anchor head train with the native loss (`anchor_loss.head_loss`): rebinds
    `AnchorBasedDetection3DHead.loss` in `visualDet3D.networks.heads.detection_3d_head`, which StereoHead (Stereo3D) and GroundAwareHead
    (Yolo3D, GroundAwareYolo3D) inherit, so the unmodified scripts/train.py computes their head loss on the GPU path.  Each call reads the
    head's own settings (num_classes, loss_cfg, focal_loss_gamma, balance_weights, regression_weight, loss_bbox.alpha).  Returns the
    installed function."""
    from visualDet3D.networks.heads import detection_3d_head as ref_head    # ImportError if the reference is not on sys.path
    from .anchor_loss import head_loss
    ref_head.AnchorBasedDetection3DHead.loss = head_loss
    return head_loss


def install_retinanet_loss_into_reference():
    """Make the REFERENCE's RetinaNet head train with the native loss (`retina_loss.head_loss`): rebinds `RetinanetHead.loss` in
    `visualDet3D.networks.heads.retinanet_head`, so the unmodified scripts/train.py (train_mono_detection) computes the 2-D detector's head
    loss on the GPU path while the reference's own RetinaNet modules compute the features.  DETECTOR_DICT is left alone:
    `install_retinanet_into_reference()` stays the inference swap.  Each call reads the head's num_clasess, loss_cfg, target_means /
    target_stds and its focal loss's gamma and balance_weights.  Returns the installed function."""
    from visualDet3D.networks.heads import retinanet_head as ref_head        # ImportError if the reference is not on sys.path
    from .retina_loss import head_loss
    ref_head.RetinanetHead.loss = head_loss
    return head_loss


def install_monoflex_loss_into_reference():
    """Make the REFERENCE's MonoFlex head train with the native loss (`monoflex_loss.head_loss`): rebinds `MonoFlexHead.loss` in
    `visualDet3D.networks.heads.monoflex_head`, so the unmodified scripts/train.py (train_rtm3d) computes MonoFlex's head loss on the GPU
    path.  KM3DHead keeps its own loss.  Each call reads the head's uncertainty_range and uncertainty_weight.  Returns the installed
    function."""
    from visualDet3D.networks.heads import monoflex_head as ref_head         # ImportError if the reference is not on sys.path
    from .monoflex_loss import head_loss
    ref_head.MonoFlexHead.loss = head_loss
    return head_loss


def install_km3d_loss_into_reference():
    """Make the REFERENCE's KM3D head train with the native loss (`km3d_loss.head_loss`): rebinds `KM3DHead.loss` in
    `visualDet3D.networks.heads.km3d_head`, so the unmodified scripts/train.py (train_rtm3d) computes KM3D's head loss on the GPU path.
    MonoFlexHead subclasses KM3DHead but defines its own loss, which stays as it is.  Each call reads the head's position_loss.output_w
    and rampup_length.  Returns the installed function."""
    from visualDet3D.networks.heads import km3d_head as ref_head             # ImportError if the reference is not on sys.path
    from .km3d_loss import head_loss
    ref_head.KM3DHead.loss = head_loss
    return head_loss


def install_disparity_loss_into_reference():
    """Make the REFERENCE's Stereo3D train its disparity branch with the native loss (`disparity_loss.forward`): rebinds
    `DisparityLoss.forward` in `visualDet3D.networks.heads.losses`, so the unmodified `Stereo3D.train_forward` (scripts/train.py,
    train_stereo_detection) computes the stereo focal loss on the GPU path.  With `install_loss_into_reference()` the whole Stereo3D
    training loss is native.  Each call reads the criterion's max_disp and refuses settings other than the shipped ones.  Returns the
    installed function."""
    from visualDet3D.networks.heads import losses as ref_losses               # ImportError if the reference is not on sys.path
    from .disparity_loss import forward
    ref_losses.DisparityLoss.forward = forward
    return forward
