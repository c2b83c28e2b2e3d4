"""Deterministic synthetic weights / priors / inputs / configs (SURVEY.md section 8(d)).

There is no network for KITTI or checkpoints, so the bench, the smoke test and the parity tests all run on
seeded synthetic data of the reference's shapes.  Every tensor is drawn from its own generator seeded by
crc32(key) so the values do not depend on state_dict iteration order: the reference module, the oracle port and
the CUDA path all see bit-identical weights.

Degenerate reference inits are re-randomised (zero-filled final cls/reg convs detection_3d_head.py:66-67,81-82,
zero DCN offset convs deform_conv.py:453-457, LookGround.alpha = 0 look_ground.py:22, identity BN stats),
otherwise parity tests would prove nothing.
"""
from __future__ import annotations

import math
import os
import zlib
from collections import OrderedDict
from typing import Dict, Mapping, Sequence, Tuple

import numpy as np
import torch

KITTI_P2 = np.array([[721.5377, 0.0, 609.5593, 44.85728],
                     [0.0, 721.5377, 172.854, 0.2163791],
                     [0.0, 0.0, 1.0, 0.002745884]], dtype=np.float64)
KITTI_HW = (375, 1242)
CROP_TOP = 100


def _gen(key: str, seed: int) -> torch.Generator:
    g = torch.Generator()
    g.manual_seed((zlib.crc32(key.encode()) ^ (seed * 0x9E3779B1)) & 0x7FFFFFFF)
    return g


CLS_GAIN = {"GroundAwareYolo3D": 3.2}     # final cls conv gain per detector kind (default 1.6): keeps ~1 % of anchors above score_thr
RETINA_CLS_BIAS = 5.0     # subtracted from the seeded retina_cls bias: tens of boxes above score_thr = 0.2 after NMS at 288x1280


def synth_state_dict(shapes: Mapping[str, Sequence[int]], seed: int = 0, gain: float = 0.8, cls_gain: float = 1.6) -> "OrderedDict[str, torch.Tensor]":
    """shapes: name -> shape for every entry of a reference-format state_dict.  Returns fp32 CPU tensors for all
    parameters and BN buffers (training-only buffers such as balance_weights are left out -> load with strict=False)."""
    names = set(shapes.keys())
    out: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    for k, shp in shapes.items():
        shp = tuple(int(s) for s in shp)
        g = _gen(k, seed)
        leaf = k.rsplit(".", 1)[-1]
        stem = k[: -len(leaf) - 1]
        is_bn = (stem + ".running_mean") in names
        if leaf == "num_batches_tracked":
            out[k] = torch.zeros(shp, dtype=torch.int64)
        elif leaf == "running_mean":
            out[k] = torch.randn(shp, generator=g) * 0.1
        elif leaf == "running_var":
            out[k] = torch.rand(shp, generator=g) + 0.5
        elif is_bn and leaf == "weight":
            w = torch.rand(shp, generator=g) + 0.5
            # last BN of a residual branch: damp, so activations stay O(1) through 16+ residual blocks
            if stem.endswith(".bn2") or stem.endswith(".bn3"):
                w = w * 0.35
            out[k] = w
        elif is_bn and leaf == "bias":
            out[k] = torch.randn(shp, generator=g) * 0.1
        elif leaf == "weight" and len(shp) >= 3:
            fan_in = int(np.prod(shp[1:]))
            std = gain * math.sqrt(2.0 / fan_in)
            if k.endswith("cls_feature_extraction.6.weight"):
                std = cls_gain / math.sqrt(fan_in)
            elif "reg_feature_extraction" in k and len(shp) == 4 and stem.rsplit(".", 1)[-1].isdigit() \
                    and _is_last_reg(k, names):
                std = 0.5 / math.sqrt(fan_in)
            elif "conv_offset" in k:
                std = 0.6 / math.sqrt(fan_in)
            elif "head_layers." in k and k.endswith(".2.weight"):      # CenterNet head outputs (zero-ish in the reference init)
                std = 1.2 / math.sqrt(fan_in)
            elif "deconv_layers." in k and len(shp) == 4 and shp[1] > 1 and shp[2:] == (4, 4):
                # dense ConvTranspose2d(4, stride 2) of the ResNet CenterNet core, [Cin, Cout, 4, 4]: every output pixel sums Cin x 2 x 2 taps
                # (not Cout x 16), so He-scale to that fan-in and the three layers keep activations O(1)
                std = gain * math.sqrt(2.0 / (shp[0] * 4))
            if (stem + ".conv_offset.weight") in names:              # DCNv2 main weights: the sigmoid mask (~0.5) halves the response
                std = std * 2.0
            if ".up_" in k and len(shp) == 4 and shp[1] == 1:          # depthwise ConvTranspose2d of IDAUp: bilinear-like, positive
                out[k] = torch.rand(shp, generator=g) * 0.2 + 0.15
                continue
            out[k] = torch.randn(shp, generator=g) * std
        elif leaf == "bias":
            b = torch.randn(shp, generator=g) * 0.05
            if k.endswith("cls_feature_extraction.6.bias"):
                b = b - 3.3
            elif k.endswith("head_layers.hm.2.bias") or k.endswith("head_layers.hm_hp.2.bias"):   # heat-map prior (km3d_head.py:146-148: -2.19)
                b = b - 3.5
            elif k.endswith("retina_cls.0.bias"):                    # RetinaNet cls prior (retinanet_head.py:66-68: log(0.01 / 0.99))
                b = b - RETINA_CLS_BIAS
            out[k] = b
        elif leaf == "alpha" and shp == (1,):            # LookGround.alpha
            out[k] = torch.full(shp, 0.5)
        elif leaf == "weight":                           # 1-D non-BN weight (e.g. Scale)
            out[k] = torch.rand(shp, generator=g) + 0.5
        # everything else (balance_weights, regression_weight ...) is a training-only buffer: skipped
    return out


def _is_last_reg(k: str, names) -> bool:
    """True for the final conv of a reg_feature_extraction Sequential (highest numeric index with a 4-D weight)."""
    stem = k[: -len(".weight")]
    head, idx = stem.rsplit(".", 1)
    best = -1
    for n in names:
        if n.startswith(head + ".") and n.endswith(".weight"):
            t = n[len(head) + 1: -len(".weight")]
            if t.isdigit():
                best = max(best, int(t))
    return int(idx) == best


def synth_priors(n_scales: int = 16, n_ratios: int = 3, obj_types: Sequence[str] = ("Car", "Pedestrian"), seed: int = 0
                 ) -> Tuple[np.ndarray, np.ndarray]:
    """anchor_{mean,std}_{type}.npy stand-ins: [types, n_scales, n_ratios, 6] float64 (z, sin2a, cos2a, w, h, l)
    in the format imdb_precompute_3d.py:63-68,165-174 writes.  A few cells carry the invalid sentinel
    (mean -100, std 1e10, :158-163) so the `z_mean > 0` filter is exercised."""
    rng = np.random.RandomState(1234 + seed)
    T = len(obj_types)
    mean = np.zeros([T, n_scales, n_ratios, 6])
    std = np.zeros([T, n_scales, n_ratios, 6])
    whl = {"Car": (1.6, 1.5, 3.9), "Pedestrian": (0.66, 1.76, 0.84), "Cyclist": (0.6, 1.7, 1.76)}
    for t, name in enumerate(obj_types):
        z = np.linspace(60.0, 4.0, n_scales)[:, None] * (1.0 + 0.08 * np.arange(n_ratios)[None, :]) * (1.0 if t == 0 else 0.8)
        mean[t, :, :, 0] = z
        std[t, :, :, 0] = 0.1 * z + 0.5
        mean[t, :, :, 1] = rng.uniform(-0.1, 0.1, [n_scales, n_ratios])
        std[t, :, :, 1] = 0.6
        mean[t, :, :, 2] = 0.3 + rng.uniform(-0.1, 0.1, [n_scales, n_ratios])
        std[t, :, :, 2] = 0.6
        w, h, l = whl.get(name, (1.0, 1.5, 2.0))
        mean[t, :, :, 3:6] = np.array([w, h, l])[None, None, :] * (1 + rng.uniform(-0.05, 0.05, [n_scales, n_ratios, 3]))
        std[t, :, :, 3:6] = np.array([0.1, 0.14, 0.43])[None, None, :]
        # invalid cells
        for (s, r) in [(0, 0), (n_scales - 1, n_ratios - 1), (3, 1 % n_ratios)]:
            if t == 1 or (s, r) != (3, 1 % n_ratios):
                mean[t, s, r, :] = -100.0
                std[t, s, r, :] = 1e10
    return mean, std


def write_priors(dirpath: str, mean: np.ndarray, std: np.ndarray, obj_types: Sequence[str]) -> str:
    """Writes {dirpath}/training/anchor_{mean,std}_{type}.npy the way Anchors.__init__ reads them (anchors.py:33-40)."""
    d = os.path.join(dirpath, "training")
    os.makedirs(d, exist_ok=True)
    for i, t in enumerate(obj_types):
        np.save(os.path.join(d, f"anchor_mean_{t}.npy"), mean[i])
        np.save(os.path.join(d, f"anchor_std_{t}.npy"), std[i])
    return dirpath


def synth_head_outputs(B: int, N: int, C: int, seed: int = 0) -> Tuple[torch.Tensor, torch.Tensor]:
    """Stand-ins for a 3-D anchor head's outputs, for the loss tests: cls [B, N, C+1] logits on a 1/8 grid over [-6, 2] and
    reg [B, N, 12] on a 1/16 grid over [-2, 2], float32 from a seeded numpy RandomState (the same values on every machine).  On that
    grid no focal-loss element lies near the reference's 1e-5 cut, so the cut decides the same way on the host and the device."""
    rng = np.random.RandomState(seed)
    cls = rng.randint(-48, 17, size=(B, N, C + 1)).astype(np.float32) / 8
    reg = rng.randint(-32, 33, size=(B, N, 12)).astype(np.float32) / 16
    return torch.from_numpy(cls), torch.from_numpy(reg)


def retina_head_outputs(B: int, N: int, C: int, seed: int = 0) -> Tuple[torch.Tensor, torch.Tensor]:
    """Stand-ins for the RetinaNet head's outputs, for the loss tests: cls [B, N, C] logits on a 1/8 grid over [-6, 2] and reg [B, N, 4]
    deltas on a 1/32 grid over [-1, 1] (decoded boxes mostly overlap their targets), float32 from a seeded numpy RandomState (the same
    values on every machine)."""
    rng = np.random.RandomState(seed)
    cls = rng.randint(-48, 17, size=(B, N, C)).astype(np.float32) / 8
    reg = rng.randint(-32, 33, size=(B, N, 4)).astype(np.float32) / 32
    return torch.from_numpy(cls), torch.from_numpy(reg)


def monoflex_head_outputs(B: int, C: int, H: int, W: int, seed: int = 0) -> dict:
    """Stand-ins for the MonoFlex head's nine output maps (fp32 NCHW), for the loss tests, from a seeded numpy RandomState (the same
    values on every machine).  hm logits lie on a 1/8 grid over [-6, 6], which keeps sigmoid well away from the focal loss's 0.99 / 0.01
    cuts; the keypoint y channels put keypoints 2, 3, 6, 7 and 8 below 0, 1, 4, 5 and 9, so the keypoint heights are mostly positive and
    the keypoint depths land inside [0.1, 100]; depth decodes (exp(-depth)) to 4..55 m."""
    rng = np.random.RandomState(seed)
    u = lambda lo, hi, ch: rng.uniform(lo, hi, size=(B, ch, H, W)).astype(np.float32)  # noqa: E731
    out = dict(hm=(rng.randint(-48, 49, size=(B, C, H, W)) / 8).astype(np.float32), bbox2d=u(0.5, 12.0, 4))
    hps = u(-10.0, 10.0, 20)
    below = np.array([-1, -1, 1, 1, -1, -1, 1, 1, 1, -1], dtype=np.float32)
    hps[:, 1::2] = below[None, :, None, None] * u(1.5, 8.0, 10)
    out.update(hps=hps, rot=u(-2.0, 2.0, 8), dim=u(1.0, 4.0, 3), reg=u(0.0, 1.0, 2), depth=u(-4.0, -1.4, 1),
               depth_uncertainty=u(-1.0, 3.0, 1), corner_uncertainty=u(-1.0, 3.0, 3))
    return {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in out.items()}


def synth_P2(B: int, H: int, W: int, seed: int = 1, jitter: float = 0.02) -> Tuple[torch.Tensor, torch.Tensor]:
    """KITTI P2 pushed through CropTop(100) + Resize((H, W)) like stereo_augmentator.py:213-258 does, with a
    per-image +-jitter on fx/fy/cy so the [B, N] useful-mask path is exercised.  P3 = P2 with Tx -= 0.54 fx."""
    rng = np.random.RandomState(seed)
    sx = W / KITTI_HW[1]
    sy = H / (KITTI_HW[0] - CROP_TOP)
    P2s, P3s = [], []
    for b in range(B):
        P = KITTI_P2.copy()
        P[1, 2] -= CROP_TOP * P[2, 2]
        P[1, 3] -= CROP_TOP * P[2, 3]
        P[0, :] *= sx
        P[1, :] *= sy
        if jitter > 0 and b > 0:
            f = 1.0 + rng.uniform(-jitter, jitter)
            P[0, 0] *= f
            P[1, 1] *= f
            P[1, 2] *= 1.0 + rng.uniform(-jitter, jitter)
        P3 = P.copy()
        P3[0, 3] -= 0.54 * P[0, 0]
        P2s.append(P)
        P3s.append(P3)
    return torch.tensor(np.stack(P2s), dtype=torch.float32), torch.tensor(np.stack(P3s), dtype=torch.float32)


def synth_stereo_inputs(B: int, H: int, W: int, seed: int = 1):
    """Post-Normalize KITTI images are ~N(0,1) (stereo_augmentator.py:39-59).  The right image is the left one
    shifted by a few pixels plus noise so the correlation volume has structure."""
    g = torch.Generator()
    g.manual_seed(seed)
    left = torch.randn(B, 3, H, W, generator=g)
    noise = torch.randn(B, 3, H, W, generator=g)
    right = 0.6 * torch.roll(left, shifts=-12, dims=3) + 0.8 * noise
    P2, P3 = synth_P2(B, H, W, seed)
    return left.contiguous(), right.contiguous(), P2, P3


def synth_mono_inputs(B: int, H: int, W: int, seed: int = 1):
    g = torch.Generator()
    g.manual_seed(seed)
    img = torch.randn(B, 3, H, W, generator=g)
    P2, _ = synth_P2(B, H, W, seed)
    return img.contiguous(), P2


class AttrDict(dict):
    """Attribute dict with the EasyDict surface the reference configs use (cfg.detector.head.anchors_cfg ...)."""

    def __init__(self, d=None, **kw):
        super().__init__()
        d = dict(d or {})
        d.update(kw)
        for k, v in d.items():
            self[k] = v

    def __setitem__(self, k, v):
        if isinstance(v, dict) and not isinstance(v, AttrDict):
            v = AttrDict(v)
        super().__setitem__(k, v)

    __setattr__ = __setitem__

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)

    def copy(self):
        return AttrDict(dict.copy(self))


def stereo3d_cfg(preprocessed_path: str, obj_types=("Car", "Pedestrian"), depth: int = 34) -> AttrDict:
    """cfg.detector of R/config/Stereo3D_example:111-167."""
    obj_types = list(obj_types)
    anchors = AttrDict(obj_types=obj_types, pyramid_levels=[4], strides=[2 ** 4], sizes=[24],
                       ratios=np.array([0.5, 1, 2.0]), scales=np.array([2 ** (i / 4.0) for i in range(16)]))
    det = AttrDict(obj_types=obj_types, name="Stereo3D")
    det.backbone = AttrDict(depth=depth, pretrained=False, frozen_stages=-1, num_stages=3, out_indices=(0, 1, 2),
                            norm_eval=True, dilations=(1, 1, 1))
    det.head = AttrDict(
        num_regression_loss_terms=13, preprocessed_path=preprocessed_path, num_classes=len(obj_types),
        anchors_cfg=anchors,
        layer_cfg=AttrDict(num_features_in=1408, num_cls_output=len(obj_types) + 1, num_reg_output=12,
                           cls_feature_size=256, reg_feature_size=1408),
        loss_cfg=AttrDict(fg_iou_threshold=0.5, bg_iou_threshold=0.4, L1_regression_alpha=5 ** 2, focal_loss_gamma=2.0,
                          balance_weight=[20.0, 40], regression_weight=[1, 1, 1, 1, 1, 1, 12, 1, 1, 0.5, 0.5, 0.5, 1]),
        test_cfg=AttrDict(score_thr=0.75, cls_agnostic=False, nms_iou_thr=0.4, post_optimization=False))
    det.anchors = anchors
    return det


def mono3d_cfg(preprocessed_path: str, kind: str = "Yolo3D", obj_types=("Car",), depth=None) -> AttrDict:
    """cfg.detector of R/config/Yolo3D_example:110-167.  kind 'GroundAwareYolo3D' = the shipped config (ResNet-101,
    1024-channel head); kind 'Yolo3D' = BASELINE.json configs[0] (ResNet-18 plumbing case: 256-channel features, DCNv2 head)."""
    obj_types = list(obj_types)
    depth = depth or (101 if kind == "GroundAwareYolo3D" else 18)
    feat = 1024 if depth > 34 else 256
    anchors = AttrDict(obj_types=obj_types, pyramid_levels=[4], strides=[2 ** 4], sizes=[24],
                       ratios=np.array([0.5, 1]), scales=np.array([2 ** (i / 4.0) for i in range(16)]))
    det = AttrDict(obj_types=obj_types, name=kind)
    det.backbone = AttrDict(depth=depth, pretrained=False, frozen_stages=-1, num_stages=3, out_indices=(2,), norm_eval=False,
                            dilations=(1, 1, 1))
    det.head = AttrDict(
        num_regression_loss_terms=13, preprocessed_path=preprocessed_path, num_classes=len(obj_types), anchors_cfg=anchors,
        layer_cfg=AttrDict(num_features_in=feat, num_cls_output=len(obj_types) + 1, num_reg_output=12,
                           cls_feature_size=feat // 2, reg_feature_size=feat),
        loss_cfg=AttrDict(fg_iou_threshold=0.5, bg_iou_threshold=0.4, L1_regression_alpha=5 ** 2, focal_loss_gamma=2.0,
                          match_low_quality=False, balance_weight=[20.0],
                          regression_weight=[1, 1, 1, 1, 1, 1, 3, 1, 1, 0.5, 0.5, 0.5, 1]),
        test_cfg=AttrDict(score_thr=0.75, cls_agnostic=False, nms_iou_thr=0.5, post_optimization=False))
    det.anchors = anchors
    return det


def retinanet_cfg(obj_types=("Car", "Pedestrian", "Cyclist"), depth: int = 50, nms_pre: int = 1000) -> AttrDict:
    """cfg.detector of R/config/RetinaNet_example (with pretrained=False: there is no network for the ImageNet weights)."""
    obj_types = list(obj_types)
    det = AttrDict(obj_types=obj_types, name="RetinaNet")
    det.backbone = AttrDict(depth=depth, pretrained=False, frozen_stages=1, num_stages=4, out_indices=(1, 2, 3), norm_eval=True)
    c = 4 if depth > 34 else 1
    det.neck = AttrDict(in_channels=[128 * c, 256 * c, 512 * c], out_channels=256, num_outs=5)
    anchors = AttrDict(pyramid_levels=[i for i in range(3, 8)], strides=[2 ** i for i in range(3, 8)], sizes=[4 * 2 ** i for i in range(3, 8)],
                       ratios=np.array([0.5, 1, 2.0]), scales=np.array([2 ** (i / 3.0) for i in range(3)]))
    det.head = AttrDict(stacked_convs=4, in_channels=256, feat_channels=256, num_classes=len(obj_types),
                        target_stds=[1.0, 1.0, 1.0, 1.0], target_means=[0.0, 0.0, 0.0, 0.0], anchors_cfg=anchors,
                        loss_cfg=AttrDict(fg_iou_threshold=0.5, bg_iou_threshold=0.4, min_iou_threshold=0, gamma=2.0, balance_weights=[1],
                                          pos_weight=-1),
                        test_cfg=AttrDict(nms_pre=nms_pre, score_thr=0.2, cls_agnostic=False, nms_iou_thr=0.4))
    return det
