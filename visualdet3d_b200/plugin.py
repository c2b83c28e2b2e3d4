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


# The reference's training datasets, the position of their images in the collate_fn's tuple, and the training function that consumes it.
_AUG_DATASETS = (("visualDet3D.data.kitti.dataset.stereo_dataset", "KittiStereoDataset", 2),
                 ("visualDet3D.data.kitti.dataset.mono_dataset", "KittiMonoDataset", 1),
                 ("visualDet3D.data.kitti.dataset.KM3D_dataset", "KittiRTM3DDataset", 1))
_AUG_TRAINERS = {"train_stereo_detection": 2, "train_mono_detection": 1, "train_rtm3d": 1}


def install_train_augmentation_into_reference():
    """Make the REFERENCE's training datasets augment on the GPU (`train_augment.TrainAugmentation`, `csrc/train_augment.cu`):
      * `build_augmentator` of the three dataset modules returns a `TrainAugmentation` for a training list it supports (one with a random
        transform; the five shipped training lists) and the reference's own `Compose` for every other list, test lists included;
      * the `collate_fn` of KittiStereoDataset, KittiMonoDataset and KittiRTM3DDataset (KittiMonoFlexDataset inherits it) stacks the
        DeferredFrames of a batch into one `train_augment.DeferredBatch` (uint8 staging + parameters; both cameras of a stereo batch in one)
        where the reference stacked float images; every other element comes from the reference's collate_fn unchanged;
      * `train_stereo_detection`, `train_mono_detection` and `train_rtm3d` in PIPELINE_DICT turn the DeferredBatch into the CUDA float
        batch (one upload, one kernel) and call the reference function unchanged.
    The numpy RNG draws are the reference's, so labels, P2 / P3 and disparity are the reference's and the images agree within the
    augmentation's parity bound (DESIGN §3.18).  Returns the installed build_augmentator."""
    import importlib
    from visualDet3D.data.pipeline import build_augmentator as ref_build     # ImportError if the reference is not on sys.path
    from visualDet3D.networks.utils import registry as ref
    from . import train_augment as ta

    def build_augmentator(aug_cfg):
        if ta.is_training_list(aug_cfg) and ta.supports(aug_cfg):
            return ta.TrainAugmentation(aug_cfg)
        return ref_build(aug_cfg)

    for modname, clsname, nimg in _AUG_DATASETS:
        mod = importlib.import_module(modname)
        mod.build_augmentator = build_augmentator
        cls = getattr(mod, clsname)
        ref_collate = getattr(cls.collate_fn, "_vd3d_ref", cls.collate_fn)           # installing twice wraps the reference once
        cls.collate_fn = staticmethod(_deferred_collate(ref_collate, nimg))

    for name, nimg in _AUG_TRAINERS.items():
        fn = ref.PIPELINE_DICT[name]
        fn = getattr(fn, "_vd3d_ref", fn)
        ref.PIPELINE_DICT._register_module(_deferred_trainer(fn, nimg), force=True)
    return build_augmentator


def install_train_targets_into_reference():
    """Make the REFERENCE's KM3D and MonoFlex datasets build their training targets on the GPU (`center_targets`,
    `csrc/center_targets.cu`):
      * `_build_target` of KittiRTM3DDataset and KittiMonoFlexDataset returns a `center_targets.DeferredTargets` (the image's packed
        labels; only `image.shape` is read, so a numpy image and a DeferredFrame both work);
      * their `collate_fn` stacks those into one `center_targets.DeferredTargetBatch` where the reference stacked the target dict;
      * `train_rtm3d` in PIPELINE_DICT turns it into the reference's target dict of CUDA tensors (one upload, two launches) and calls the
        reference function unchanged, whose `gts[key].cuda()` is then a no-op.
    Works alone and with `install_train_augmentation_into_reference()`, in either order.  Returns the installed `_build_target`."""
    from visualDet3D.data.kitti.dataset import KM3D_dataset as mod              # ImportError if the reference is not on sys.path
    from visualDet3D.networks.utils import registry as ref
    from . import center_targets as ct

    def _build_target(self, image, P2, transformed_label, scale=4):
        if scale != ct.SCALE:
            raise NotImplementedError(f"_build_target: the GPU targets use the reference's scale {ct.SCALE}, not {scale}")
        mode = {9: ct.MODE_KM3D, 10: ct.MODE_MONOFLEX}[self.num_vertexes]
        return ct.DeferredTargets.build(image.shape, P2, transformed_label, [self.obj_types.index(o.type) for o in transformed_label],
                                        self.num_classes, mode)

    mod.KittiRTM3DDataset._build_target = _build_target
    mod.KittiMonoFlexDataset._build_target = _build_target
    cls = mod.KittiRTM3DDataset
    cls.collate_fn = staticmethod(_deferred_collate(getattr(cls.collate_fn, "_vd3d_ref", cls.collate_fn), 1))
    fn = ref.PIPELINE_DICT["train_rtm3d"]
    ref.PIPELINE_DICT._register_module(_deferred_trainer(getattr(fn, "_vd3d_ref", fn), 1), force=True)
    return _build_target


# The position of the target dict in the KM3D / MonoFlex collate_fn's (images, calib, label) tuple.
_TARGET_SLOT = 2


def _deferred_collate(ref_collate, nimg):
    """The collate_fn of both training installs: DeferredFrames become one DeferredBatch (install_train_augmentation_into_reference) and
    DeferredTargets one DeferredTargetBatch (install_train_targets_into_reference); everything else comes from the reference's."""
    import numpy as np
    from .center_targets import DeferredTargetBatch, DeferredTargets
    from .train_augment import DeferredBatch, DeferredFrame

    def collate_fn(batch):
        first = batch[0]["image"]
        images = isinstance(first[0] if nimg == 2 else first, DeferredFrame)
        targets = isinstance(batch[0].get("label"), DeferredTargets)
        if not (images or targets):
            return ref_collate(batch)
        tiny = np.zeros((1, 1, 3), np.float32)           # the reference stacks these in place of the images; its other outputs are kept
        stub = {}
        if images:
            stub["image"] = [tiny, tiny] if nimg == 2 else tiny
        if targets:
            stub["label"] = {}                           # an empty target dict collates to {}
        out = list(ref_collate([dict(item, **stub) for item in batch]))
        if images:
            frames = [item["image"][0] for item in batch] + [item["image"][1] for item in batch] if nimg == 2 else \
                [item["image"] for item in batch]
            out[:nimg] = [DeferredBatch(frames)] * nimg
        if targets:
            out[_TARGET_SLOT] = DeferredTargetBatch([item["label"] for item in batch])
        return tuple(out)

    collate_fn._vd3d_ref = ref_collate
    collate_fn.__name__ = "collate_fn"
    return collate_fn


def _deferred_trainer(ref_fn, nimg):
    import functools
    from .center_targets import DeferredTargetBatch
    from .train_augment import DeferredBatch

    @functools.wraps(ref_fn)
    def train(data, *args, **kwargs):
        if ref_fn.__name__ == "train_rtm3d" and isinstance(data[_TARGET_SLOT], DeferredTargetBatch):
            data = tuple(data[:_TARGET_SLOT]) + (data[_TARGET_SLOT].to_device("cuda"),) + tuple(data[_TARGET_SLOT + 1:])
        if isinstance(data[0], DeferredBatch):
            images = data[0].to_device("cuda")
            B = len(data[0]) // nimg
            data = list(data)
            data[:nimg] = [images[:B], images[B:]] if nimg == 2 else [images]
            if ref_fn.__name__ == "train_rtm3d":
                data[1] = data[1].cuda()                 # `image.new(K)` aliases K: it must be on the images' device
            data = tuple(data)
        return ref_fn(data, *args, **kwargs)

    train._vd3d_ref = ref_fn
    return train
