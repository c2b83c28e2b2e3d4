"""ORACLE (test infrastructure, not product code): KM3D / MonoFlex with the ResNet CenterNet core, in plain fp32 PyTorch on the CPU.

oracle/torch_port.py covers the DLA-34 core.  This module adds the other core of KM3DCore (R/detectors/KM3D_core.py:34-58), the one
KM3D_example builds: a ResNet whose last returned map goes through three ConvTranspose2d(4, stride 2, padding 1, no bias) + BN + ReLU.
Everything after the core is torch_port's own (heads, decodes), so the two oracles share their decode arithmetic.  Pinned against the
unmodified reference by tests/golden/make_golden_km3d_resnet.py and tests/test_km3d_resnet_cpu.py.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

import torch_port as tp


def resnet_core(sd: tp.SD, images, backbone_cfg: dict):
    """KM3DCore.forward for a ResNet backbone (KM3D_core.py:52-58): deconv_layers(backbone(image)[-1]) -> (features, backbone outputs)."""
    ys = tp.resnet(sd, "core.backbone", images, int(backbone_cfg["depth"]), int(backbone_cfg.get("num_stages", 4)),
                   tuple(backbone_cfg.get("out_indices", (-1, 0, 1, 2, 3))), tuple(backbone_cfg.get("strides", (1, 2, 2, 2))),
                   tuple(backbone_cfg.get("dilations", (1, 1, 1, 1))))
    x = ys[-1]
    for i in (0, 3, 6):
        x = F.conv_transpose2d(x, sd[f"core.deconv_layers.{i}.weight"], None, stride=2, padding=1)
        x = F.relu(tp.bn(sd, f"core.deconv_layers.{i + 1}", x))
    return x, ys


def monoflex_forward(sd: tp.SD, images, P2, cfg: dict, stages: dict | None = None):
    """MonoFlex.test_forward (R/detectors/KM3D.py:61-79) on the ResNet core, decode looped per image (torch_port.monoflex_get_bboxes)."""
    with torch.no_grad():
        feat, ys = resnet_core(sd, images, cfg["backbone"])
        outs = tp.km3d_heads(sd, feat, list(cfg["head"]["layer_cfg"]["head_dict"].keys()))
        if stages is not None:
            stages.update(features=feat, heads=outs, levels=ys)
        tc = cfg["head"]["test_cfg"]
        return [tp.monoflex_get_bboxes({k: v[b:b + 1] for k, v in outs.items()}, P2[b:b + 1], images.shape[2:], tc.get("score_thr", 0.1),
                                       tc.get("nms_iou_thr", 0.5))
                for b in range(images.shape[0])]


def km3d_forward(sd: tp.SD, images, P2, cfg: dict, stages: dict | None = None):
    """KM3D.test_forward (R/detectors/KM3D.py:61-79) on the ResNet core, decode looped per image (torch_port.km3d_get_bboxes)."""
    with torch.no_grad():
        feat, _ = resnet_core(sd, images, cfg["backbone"])
        outs = tp.km3d_heads(sd, feat, list(cfg["head"]["layer_cfg"]["head_dict"].keys()))
        if stages is not None:
            stages.update(features=feat, heads=outs)
        tc = cfg["head"]["test_cfg"]
        return [tp.km3d_get_bboxes({k: v[b:b + 1] for k, v in outs.items()}, P2[b:b + 1], images.shape[2:], tc.get("score_thr", 0.1),
                                   tc.get("nms_iou_thr", 0.5))
                for b in range(images.shape[0])]
