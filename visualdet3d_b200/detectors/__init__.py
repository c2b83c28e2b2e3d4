"""Detectors registered under the reference's names in `visualdet3d_b200.plugin.DETECTOR_DICT`."""
from .stereo3d import Stereo3D, build_synthetic_stereo3d  # noqa: F401
from .mono3d import Yolo3D, GroundAwareYolo3D, build_synthetic_mono3d  # noqa: F401
from .centernet import MonoFlex, KM3D, build_synthetic_monoflex, monoflex_cfg, km3d_cfg, km3d_example_cfg, monoflex_resnet_cfg  # noqa: F401
from .retinanet import RetinaNet, build_synthetic_retinanet  # noqa: F401
