"""Parameter-holder module trees that reproduce the reference's ``state_dict`` key names.

The scripts treat a detector as an ``nn.Module`` (``.cuda()``, ``.eval()``, ``.load_state_dict``, ``.parameters()``,
``SyncBatchNorm.convert`` ... SURVEY.md section 8(b)), and checkpoints are keyed by the reference's attribute paths
(e.g. ``core.neck.depth_reasoning.four_to_eight.0.primary_conv.1.weight``).  These classes own real
``nn.Parameter``s under exactly those paths.  They are never *executed* by torch on the B200 path: the engine folds
the parameters into packed device weights and launches libvd3d_b200 kernels.  Calling ``forward`` on a holder raises.
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn


class Holder(nn.Module):
    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("parameter holder: the B200 path executes through visualdet3d_b200.engine, not torch ops")


def seq(*mods) -> nn.Sequential:
    return nn.Sequential(*mods)


class BasicBlockP(Holder):
    """keys of R/backbones/resnet.py:23-35."""
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=None, dilation=1):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 3, stride, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, 3, 1, dilation, dilation=dilation, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.downsample = downsample
        self.stride, self.dilation = stride, dilation


class BottleneckP(Holder):
    """keys of R/backbones/resnet.py:55-71."""
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None, dilation=1):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, 3, stride, dilation, dilation=dilation, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, planes * 4, 1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.downsample = downsample
        self.stride, self.dilation = stride, dilation


RESNET_SPECS = {18: (BasicBlockP, (2, 2, 2, 2)), 34: (BasicBlockP, (3, 4, 6, 3)), 50: (BottleneckP, (3, 4, 6, 3)),
                101: (BottleneckP, (3, 4, 23, 3)), 152: (BottleneckP, (3, 8, 36, 3))}


class ResNetP(Holder):
    """keys of R/backbones/resnet.py:95-152; accepts the reference's backbone cfg (depth, pretrained, frozen_stages,
    num_stages, out_indices, norm_eval, dilations, strides)."""

    def __init__(self, depth, pretrained=False, num_stages=4, strides=(1, 2, 2, 2), dilations=(1, 1, 1, 1),
                 out_indices=(-1, 0, 1, 2, 3), frozen_stages=-1, norm_eval=True, **_):
        super().__init__()
        if depth not in RESNET_SPECS:
            raise ValueError("Unsupported model depth, must be one of 18, 34, 50, 101, 152")
        if pretrained:
            raise RuntimeError("pretrained=True needs a network download (resnet.py:208-209); load a checkpoint instead")
        block, layers = RESNET_SPECS[depth]
        assert 1 <= num_stages <= 4 and max(out_indices) < num_stages
        self.depth, self.block, self.layers = depth, block, layers
        self.num_stages, self.strides, self.dilations, self.out_indices = num_stages, tuple(strides), tuple(dilations), tuple(out_indices)
        self.conv1 = nn.Conv2d(3, 64, 7, 2, 3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        inplanes = 64
        for i in range(num_stages):
            planes = 64 * 2 ** i
            blocks = []
            for j in range(layers[i]):
                stride = self.strides[i] if j == 0 else 1
                ds = None
                if j == 0 and (stride != 1 or inplanes != planes * block.expansion):
                    ds = seq(nn.Conv2d(inplanes, planes * block.expansion, 1, stride, bias=False), nn.BatchNorm2d(planes * block.expansion))
                blocks.append(block(inplanes, planes, stride, ds, dilation=1 if j == 0 else self.dilations[i]))
                inplanes = planes * block.expansion
            setattr(self, f"layer{i + 1}", seq(*blocks))
        for m in self.modules():          # same init statistics as resnet.py:125-131
            if isinstance(m, nn.Conv2d):
                n = m.kernel_size[0] * m.kernel_size[1] * m.out_channels
                m.weight.data.normal_(0, math.sqrt(2.0 / n))

    def out_channels(self, stage: int) -> int:
        return 64 * 2 ** stage * self.block.expansion


class GhostP(Holder):
    """keys of R/lib/ghost_module.py:20-38 as instantiated by ResGhostModule(inp, oup, k, ratio) (:46-55)."""

    def __init__(self, inp, oup, kernel_size=3, ratio=3, dw_size=3):
        super().__init__()
        assert ratio > 2
        g_oup, g_ratio = oup - inp, ratio - 1
        init = math.ceil(g_oup / g_ratio)
        new = init * (g_ratio - 1)
        self.inp, self.oup, self.init_channels, self.new_channels, self.kernel_size = inp, oup, init, new, kernel_size
        self.primary_conv = seq(seq(), nn.Conv2d(inp, init, kernel_size, 1, kernel_size // 2, bias=False), nn.BatchNorm2d(init), nn.ReLU(inplace=True))
        self.cheap_operation = seq(nn.Conv2d(init, new, dw_size, 1, dw_size // 2, groups=init, bias=False), nn.BatchNorm2d(new), nn.ReLU(inplace=True))


class PSMCosineP(Holder):
    """R/lib/PSM_cost_volume.py:66-73 (no parameters)."""

    def __init__(self, max_disp, downsample_scale, input_features):
        super().__init__()
        self.max_disp, self.downsample_scale = max_disp, downsample_scale
        self.depth_channel = int(max_disp / downsample_scale)


class CostVolumeP(Holder):
    """keys of R/lib/PSM_cost_volume.py:20-38."""

    def __init__(self, max_disp=192, downsample_scale=4, input_features=1024, PSM_features=64):
        super().__init__()
        self.depth_channel = int(max_disp / downsample_scale)
        self.PSM_features = PSM_features
        self.down_sample = seq(nn.Conv2d(input_features, PSM_features, 1), nn.BatchNorm2d(PSM_features), nn.ReLU())
        self.conv3d = seq(nn.Conv3d(2 * PSM_features, PSM_features, 3, padding=1), nn.BatchNorm3d(PSM_features), nn.ReLU(),
                          nn.Conv3d(PSM_features, PSM_features, 3, padding=1), nn.BatchNorm3d(PSM_features), nn.ReLU())
        self.output_channel = PSM_features * self.depth_channel


class CostVolumePyramidP(Holder):
    """keys of R/detectors/yolostereo3d_core.py:16-60 (depth_output is training-only but lives in checkpoints)."""

    def __init__(self, c4, c8, c16):
        super().__init__()
        f = c4
        self.four_to_eight = seq(GhostP(f, 3 * f), nn.AvgPool2d(2), BasicBlockP(3 * f, 3 * f))
        f = 3 * f + c8
        self.eight_to_sixteen = seq(GhostP(f, 3 * f), nn.AvgPool2d(2), BasicBlockP(3 * f, 3 * f))
        f = 3 * f + c16
        self.depth_reason = seq(GhostP(f, 3 * f), BasicBlockP(3 * f, 3 * f))
        self.output_channel_num = o = 3 * f
        self.depth_output = seq(nn.Upsample(scale_factor=2, mode="bilinear", align_corners=True),
                                nn.Conv2d(o, o // 2, 3, padding=1), nn.BatchNorm2d(o // 2), nn.ReLU(),
                                nn.Upsample(scale_factor=2, mode="bilinear", align_corners=True),
                                nn.Conv2d(o // 2, o // 4, 3, padding=1), nn.BatchNorm2d(o // 4), nn.ReLU(),
                                nn.Conv2d(o // 4, 96, 1))


class StereoMergingP(Holder):
    """keys of R/detectors/yolostereo3d_core.py:73-86."""

    def __init__(self, base_features):
        super().__init__()
        self.cost_volume_0 = PSMCosineP(96, 4, base_features)
        self.cost_volume_1 = PSMCosineP(192, 8, base_features * 2)
        self.cost_volume_2 = CostVolumeP(192, 16, base_features * 4, PSM_features=8)
        self.depth_reasoning = CostVolumePyramidP(self.cost_volume_0.depth_channel, self.cost_volume_1.depth_channel,
                                                  self.cost_volume_2.output_channel)
        self.final_channel = self.depth_reasoning.output_channel_num + base_features * 4


class YoloStereo3DCoreP(Holder):
    """keys of R/detectors/yolostereo3d_core.py:96-108."""

    def __init__(self, backbone_arguments):
        super().__init__()
        self.backbone = ResNetP(**backbone_arguments)
        self.neck = StereoMergingP(256 if backbone_arguments["depth"] > 34 else 64)


class ConvBnReLUP(Holder):
    """keys of R/lib/blocks.py:24-36 (`sequence.0` conv with bias, `sequence.1` BN)."""

    def __init__(self, cin, cout, k=3):
        super().__init__()
        self.sequence = seq(nn.Conv2d(cin, cout, k, 1, (k - 1) // 2), nn.BatchNorm2d(cout))


class LossClsP(Holder):
    def __init__(self, balance_weights):
        super().__init__()
        self.register_buffer("balance_weights", balance_weights.clone())


class HeadBaseP(Holder):
    """Buffers every AnchorBasedDetection3DHead checkpoint carries (R/heads/detection_3d_head.py:90-99)."""

    def __init__(self, loss_cfg, num_regression_loss_terms):
        super().__init__()
        bw = torch.tensor(list(loss_cfg.get("balance_weight", [0])), dtype=torch.float32)
        self.register_buffer("balance_weights", bw)
        self.register_buffer("regression_weight", torch.tensor(
            list(loss_cfg.get("regression_weight", [1 for _ in range(num_regression_loss_terms)])), dtype=torch.float))
        self.loss_cls = LossClsP(bw)


def cls_tower(cin, feat, nout):
    """R/heads/detection_3d_head.py:55-65 / :509-519 (Dropout2d(0.3) is identity in eval)."""
    return seq(nn.Conv2d(cin, feat, 3, padding=1), nn.Dropout2d(0.3), nn.ReLU(inplace=True),
               nn.Conv2d(feat, feat, 3, padding=1), nn.Dropout2d(0.3), nn.ReLU(inplace=True),
               nn.Conv2d(feat, nout, 3, padding=1), nn.Identity())


class StereoHeadP(HeadBaseP):
    """keys of R/heads/detection_3d_head.py:500-533 (StereoHead.init_layers)."""

    def __init__(self, num_features_in, num_anchors, num_cls_output, num_reg_output, cls_feature_size=1024,
                 reg_feature_size=1024, loss_cfg=None, num_regression_loss_terms=12, **_):
        super().__init__(loss_cfg or {}, num_regression_loss_terms)
        self.cls_feature_extraction = cls_tower(num_features_in, cls_feature_size, num_anchors * num_cls_output)
        self.reg_feature_extraction = seq(ConvBnReLUP(num_features_in, reg_feature_size, 3),
                                          BasicBlockP(reg_feature_size, reg_feature_size), nn.ReLU(),
                                          nn.Conv2d(reg_feature_size, num_anchors * num_reg_output, 3, padding=1), nn.Identity())


class DCNPackP(Holder):
    """keys of ModulatedDeformConvPack (R/lib/ops/dcn/deform_conv.py:408-457): weight, bias, conv_offset.{weight,bias}."""

    def __init__(self, cin, cout, k=3, stride=1, padding=1, dilation=1, deformable_groups=1, bias=True):
        super().__init__()
        self.cin, self.cout, self.k = cin, cout, k
        self.stride, self.padding, self.dilation, self.deformable_groups = stride, padding, dilation, deformable_groups
        self.weight = nn.Parameter(torch.empty(cout, cin, k, k).uniform_(-1, 1) / math.sqrt(cin * k * k))
        self.bias = nn.Parameter(torch.zeros(cout)) if bias else None
        self.conv_offset = nn.Conv2d(cin, deformable_groups * 3 * k * k, k, stride, padding, bias=True)
        nn.init.zeros_(self.conv_offset.weight)
        nn.init.zeros_(self.conv_offset.bias)


class MonoHeadP(HeadBaseP):
    """keys of AnchorBasedDetection3DHead.init_layers (R/heads/detection_3d_head.py:47-82): DCNv2 reg tower."""

    def __init__(self, num_features_in, num_anchors, num_cls_output, num_reg_output, cls_feature_size=1024,
                 reg_feature_size=1024, loss_cfg=None, num_regression_loss_terms=12, **_):
        super().__init__(loss_cfg or {}, num_regression_loss_terms)
        self.cls_feature_extraction = cls_tower(num_features_in, cls_feature_size, num_anchors * num_cls_output)
        self.reg_feature_extraction = seq(DCNPackP(num_features_in, reg_feature_size, 3, padding=1), nn.BatchNorm2d(reg_feature_size),
                                          nn.ReLU(inplace=True), nn.Conv2d(reg_feature_size, reg_feature_size, 3, padding=1),
                                          nn.BatchNorm2d(reg_feature_size), nn.ReLU(inplace=True),
                                          nn.Conv2d(reg_feature_size, num_anchors * num_reg_output, 3, padding=1), nn.Identity())


class LookGroundP(Holder):
    """keys of LookGround (R/lib/look_ground.py:13-22): disp_create.0.{weight,bias}, extract.{weight,bias}, alpha."""

    def __init__(self, input_features, baseline=0.54, relative_elevation=1.65):
        super().__init__()
        self.disp_create = seq(nn.Conv2d(input_features, 1, 3, padding=1), nn.Tanh())
        self.extract = nn.Conv2d(1 + input_features, input_features, 1)
        self.baseline, self.relative_elevation = baseline, relative_elevation
        self.alpha = nn.Parameter(torch.tensor([0.0], dtype=torch.float32))


class GroundAwareHeadP(HeadBaseP):
    """keys of GroundAwareHead.init_layers (R/detectors/yolomono3d_detector.py:12-47)."""

    def __init__(self, num_features_in, num_anchors, num_cls_output, num_reg_output, cls_feature_size=1024,
                 reg_feature_size=1024, loss_cfg=None, num_regression_loss_terms=12, **_):
        super().__init__(loss_cfg or {}, num_regression_loss_terms)
        self.cls_feature_extraction = cls_tower(num_features_in, cls_feature_size, num_anchors * num_cls_output)
        self.reg_feature_extraction = seq(LookGroundP(reg_feature_size), nn.Conv2d(num_features_in, reg_feature_size, 3, padding=1),
                                          nn.BatchNorm2d(reg_feature_size), nn.ReLU(),
                                          nn.Conv2d(reg_feature_size, reg_feature_size, 3, padding=1), nn.BatchNorm2d(reg_feature_size),
                                          nn.ReLU(inplace=True), nn.Conv2d(reg_feature_size, num_anchors * num_reg_output, 3, padding=1),
                                          nn.Identity())


class YoloMono3DCoreP(Holder):
    """keys of YoloMono3DCore (R/detectors/yolomono3d_core.py:9-18)."""

    def __init__(self, backbone_arguments):
        super().__init__()
        self.backbone = ResNetP(**backbone_arguments)


class FPNP(Holder):
    """keys of FPN (R/detectors/retinanet_2d.py:15-40): lateral_convs.i (1x1, bias), fpn_convs.i (3x3, bias; the extra levels stride 2)."""

    def __init__(self, in_channels, out_channels, num_outs):
        super().__init__()
        self.in_channels, self.out_channels, self.num_outs = list(in_channels), int(out_channels), int(num_outs)
        self.lateral_convs = nn.ModuleList([nn.Conv2d(c, out_channels, 1) for c in in_channels])
        self.fpn_convs = nn.ModuleList([nn.Conv2d(out_channels, out_channels, 3, padding=1) for _ in in_channels])
        for i in range(num_outs - len(in_channels)):
            self.fpn_convs.append(nn.Conv2d(in_channels[-1] if i == 0 else out_channels, out_channels, 3, padding=1, stride=2))


class RetinaNetCoreP(Holder):
    """keys of RetinaNetCore (R/detectors/retinanet_2d.py:69-73)."""

    def __init__(self, backbone_cfg, neck_cfg):
        super().__init__()
        self.backbone = ResNetP(**backbone_cfg)
        self.neck = FPNP(**neck_cfg)


class ConvReLUP(Holder):
    """keys of ConvReLU (R/lib/blocks.py:46-60): `sequence.0` conv with bias, `sequence.1` ReLU."""

    def __init__(self, cin, cout, k=3):
        super().__init__()
        self.sequence = seq(nn.Conv2d(cin, cout, k, 1, (k - 1) // 2), nn.ReLU())


class RetinaHeadP(Holder):
    """keys of RetinanetHead (R/heads/retinanet_head.py:13-80): cls_conv / reg_conv towers, retina_cls / retina_reg (AnchorFlatten has no
    parameters), the focal-loss balance_weights buffers."""

    def __init__(self, num_anchors, stacked_convs=4, in_channels=256, feat_channels=256, num_classes=3, reg_output=4, loss_cfg=None):
        super().__init__()
        cins = [in_channels] + [feat_channels] * (stacked_convs - 1) if stacked_convs > 0 else []
        self.cls_conv = seq(*[ConvReLUP(c, feat_channels) for c in cins])
        self.reg_conv = seq(*[ConvReLUP(c, feat_channels) for c in cins])
        self.retina_cls = seq(nn.Conv2d(feat_channels, num_anchors * num_classes, 3, padding=1))
        self.retina_reg = seq(nn.Conv2d(feat_channels, num_anchors * reg_output, 3, padding=1))
        bw = torch.tensor((loss_cfg or {}).get("balance_weights", 0), dtype=torch.float32)
        self.register_buffer("balance_weights", bw)
        self.loss_cls = LossClsP(bw)
