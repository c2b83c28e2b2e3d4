"""`MonoFlex` / `KM3D` — DLA-34 + DCNv2 up-sampling, or ResNet-18 / 34 + three transposed convs, + CenterNet-style heads on the GPU
(drop-ins for R/detectors/KM3D.py:16-96, core R/detectors/KM3D_core.py:10-58, heads R/heads/km3d_head.py, monoflex_head.py).

Protocol: ``module([image[1,3,H,W], P2[1,3,4]])`` -> ``(scores[K], bboxes[K,11], cls[K])``; a 3-element list is the training
protocol (raises).  ``forward_batch(images, P2)`` runs B images at once.

Head execution: the nine `conv3x3(64->256)+ReLU` stems are ONE wgmma conv (64 -> 9*256, weights concatenated), the nine 1x1
output convs write their channel slices of one [B,H/4,W/4,56] tensor that the decode kernels gather from.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .. import engine as E
from .. import _lib
from .._lib import Vd3dError, call
from ..plugin import DETECTOR_DICT
from . import modules as M
from .base import NativeDetector, synth_load
from .dla import DLAP, DLARunner, DLASegUpsampleP, DLAUpRunner
from .stereo3d import ResNetRunner


def _peak_capacity(n_cells: int) -> int:
    """Capacity of a heat-map peak list: a 3x3 local maximum rules out its 8 neighbours, so a map of n cells has at most ~n / 4 peaks;
    power of two in [1024, 8192] (the library's limit: more peaks than that are reported as an overflow, never truncated).  The decode
    kernels sort only the occupied part of a list, so a generous capacity costs memory, not time."""
    cap = 1024
    while cap < min(8192, (n_cells + 3) // 4):
        cap <<= 1
    return cap


class KM3DCoreP(M.Holder):
    """keys of KM3DCore (R/detectors/KM3D_core.py:10-50).  The backbone follows the reference's `build_backbone`
    (R/backbones/__init__.py:5-13): `name` missing means 'resnet'.
      * 'dla' / 'dlanet' (Monoflex_example): DLA-34, then DLASegUpsample (DCNv2 IDAUp) to 64 channels at 1/4 resolution.
      * 'resnet' (KM3D_example, which names no backbone; Monoflex_example's commented-out alternative): ResNet-18 / 34 whose last stage
        (512 channels at 1/32) feeds the "baseline" up-sampling `deconv_layers` = three ConvTranspose2d(4, stride 2, padding 1, no bias)
        + BatchNorm2d + ReLU, 512 -> 256 -> 256 -> 256, to 1/4 resolution (KM3D_core.py:34-47).
    The reference's own KM3DCore reads backbone_arguments['name'] directly, so it needs the name spelled out; a name-less config builds
    here exactly what it builds with name='resnet'.  ResNet deeper than 34 is refused: the reference wires 2024 input channels into the
    first transposed conv for it (KM3D_core.py:19-20), which cannot take the 2048-channel last stage."""

    def __init__(self, backbone_arguments):
        super().__init__()
        args = dict(backbone_arguments)
        name = str(args.get("name", "resnet")).lower()
        self.backbone_name = "resnet" if name == "resnet" else "dla"
        if name in ("dla", "dlanet"):
            self.backbone = DLAP(**args)
            self.deconv_layers = DLASegUpsampleP(input_channels=[16, 32, 64, 128, 256, 512], down_ratio=4, final_kernel=1, last_level=5, out_channel=64)
        elif name == "resnet":
            args.pop("name", None)
            depth = int(args.get("depth", 0))
            if depth > 34:
                raise ValueError(f"KM3DCore with ResNet-{depth}: the reference's core gives the first transposed conv 2024 input channels "
                                 "for depth > 34 (KM3D_core.py:19-20) and cannot run the 2048-channel last stage; use depth 18 or 34")
            out_indices = tuple(args.get("out_indices", (-1, 0, 1, 2, 3)))
            if not out_indices or out_indices[-1] != 3:
                raise ValueError(f"KM3DCore with ResNet: the last out_indices entry must be stage 3 (the core up-samples the last returned "
                                 f"map, which must be the 512-channel stage 3), got {out_indices}")
            self.backbone = M.ResNetP(**args)
            feat = 256
            self.deconv_layers = M.seq(
                nn.ConvTranspose2d(self.backbone.out_channels(3), feat, 4, stride=2, padding=1, bias=False), nn.BatchNorm2d(feat), nn.ReLU(inplace=True),
                nn.ConvTranspose2d(feat, feat, 4, stride=2, padding=1, bias=False), nn.BatchNorm2d(feat), nn.ReLU(inplace=True),
                nn.ConvTranspose2d(feat, feat, 4, stride=2, padding=1, bias=False), nn.BatchNorm2d(feat), nn.ReLU(inplace=True))
        else:
            raise NotImplementedError(f"KM3DCore on the native path takes the DLA-34 or ResNet-18 / 34 backbone, not {name!r}")
        for m in self.deconv_layers.modules():
            if isinstance(m, nn.ConvTranspose2d):
                nn.init.normal_(m.weight, std=0.001)


class KM3DHeadP(M.Holder):
    """keys of KM3DHead (R/heads/km3d_head.py:23-41,132-153): buffer `const`, head_layers.<name>.{0,2}.{weight,bias}."""

    def __init__(self, num_classes=3, num_joints=9, max_objects=32, layer_cfg=None, loss_cfg=None, test_cfg=None, with_position_loss=False):
        super().__init__()
        lc = dict(layer_cfg or {})
        cin, feat = lc.get("input_features", 256), lc.get("head_features", 64)
        self.head_dict = dict(lc.get("head_dict", {}))
        self.head_layers = nn.ModuleDict()
        for name, n_out in self.head_dict.items():
            self.head_layers[name] = M.seq(nn.Conv2d(cin, feat, 3, padding=1, bias=True), nn.ReLU(inplace=True), nn.Conv2d(feat, n_out, 1))
            last = self.head_layers[name][-1]
            if "hm" in name:
                nn.init.constant_(last.bias, -2.19)
            else:
                nn.init.normal_(last.weight, std=0.001)
                nn.init.constant_(last.bias, 0)
        const = torch.tensor([[-1, 0], [0, -1]] * 8, dtype=torch.float32).unsqueeze(0).unsqueeze(0)
        self.register_buffer("const", const)
        if with_position_loss:        # KM3DHead.build_loss registers Position_loss (buffer `const`, rtm3d_utils.py:230-240); MonoFlexHead does not
            self.position_loss = M.Holder()
            self.position_loss.register_buffer("const", const.clone())
        self.num_classes, self.num_joints, self.max_objects = num_classes, num_joints, max_objects
        self.input_features, self.head_features = cin, feat


class _CenterNetBase(NativeDetector):
    """Subclasses name the decode entry (`DECODE`, `WORKSPACE`), the head maps it reads (`REQUIRED`, in the entry's argument order), the
    peak-list capacities and the decode's own scalar arguments."""
    WITH_POSITION_LOSS = False
    DECODE = WORKSPACE = None
    REQUIRED = ()

    def __init__(self, network_cfg):
        super().__init__()
        self.obj_types = network_cfg["obj_types"]
        head = network_cfg["head"]
        self.test_cfg = dict(head.get("test_cfg", {}))
        self.bbox_head = KM3DHeadP(head.get("num_classes", 3), head.get("num_joints", 9), head.get("max_objects", 32),
                                   head.get("layer_cfg", {}), head.get("loss_cfg", {}), self.test_cfg, self.WITH_POSITION_LOSS)
        self.core = KM3DCoreP(dict(network_cfg["backbone"]))
        self.network_cfg = network_cfg
        lc = dict(head.get("loss_cfg", {}))
        self.uncertainty_range = tuple(lc.get("uncertainty_range", [-10, 10]))
        self.num_classes = self.bbox_head.num_classes
        self.topk = 100

    def build_plan(self, dev) -> dict:
        if self.core.backbone_name == "resnet":
            dl = self.core.deconv_layers
            pl = dict(resnet=ResNetRunner(self.core.backbone, dev),
                      deconv=[E.ConvTransposeLayer(dl[i].weight, E.bn_dict(dl[i + 1]), relu=True, device=dev) for i in (0, 3, 6)])
        else:
            pl = dict(dla=DLARunner(self.core.backbone, dev, first_used_level=self.core.deconv_layers.first_level),
                      up=DLAUpRunner(self.core.deconv_layers, dev))
        hl = self.bbox_head.head_layers
        names = list(hl.keys())
        # one stem conv for all heads: weights / biases concatenated along Cout
        w = torch.cat([hl[n][0].weight.detach() for n in names], 0)
        b = torch.cat([hl[n][0].bias.detach() for n in names], 0)
        pl["stem"] = E.ConvLayer(w, b, None, pad=1, relu=True, device=dev)
        feat = self.bbox_head.head_features
        outs, off, co = {}, {}, 0
        # the nine 1x1 output convs (256 -> n, n = 1..20): on the tensor cores when the engine is there (n padded to 16 columns with zero
        # filters), reading the fp16 planes of their 256-channel slice of the stem output; the SIMT engine re-read 252 MB of fp32 per head
        tc_out = pl["stem"].engine == "tc16"
        gran = 16 if tc_out else 4
        for i, n in enumerate(names):
            n_out = hl[n][2].weight.shape[0]
            n_pad = (n_out + gran - 1) // gran * gran
            wo = torch.zeros(n_pad, feat, 1, 1)
            wo[:n_out] = hl[n][2].weight.detach().cpu()
            bo = torch.zeros(n_pad)
            bo[:n_out] = hl[n][2].bias.detach().cpu()
            outs[n] = (E.ConvLayer(wo, bo, None, relu=False, device=dev, engine=None if tc_out else "simt"), i * feat, co, n_pad)
            off[n] = co
            co += n_pad
        pl["outs"], pl["offsets"], pl["out_channels"], pl["names"] = outs, off, co, names
        return pl

    def network(self, images: torch.Tensor) -> E.Act:
        """core (DLA + up-sampling) + heads -> one NHWC tensor [B, H/4, W/4, out_channels] holding every head output."""
        pl = self.prepare()
        ar = self._arena
        B, _, H, W = images.shape
        if H % 32 or W % 32:
            raise Vd3dError(f"{type(self).__name__}: image size {H}x{W} must be a multiple of 32 (the backbone has 5 stride-2 levels)")
        if "resnet" in pl:
            feat = self._resnet_core(pl, images, ar)      # [B, H/4, W/4, 256]
        else:
            ys = pl["dla"].run(images, ar)
            feat = pl["up"].run(ys, ar)                   # [B, H/4, W/4, 64]
        self._hook("features", feat)
        dev = images.device
        if pl["stem"].engine != "simt":
            E.split_lo_if_stale(feat)
        tc_out = all(l.engine == "tc16" for (l, _, _, _) in pl["outs"].values())
        # the stem output (9 x 256 channels at 1/4 resolution: the largest tensor of the network) feeds only the 1x1 output convs: with
        # those on the tensor cores it is written as fp16 planes only (no fp32 copy: 2.3 GB less HBM traffic per batch-8 step at 384x1280)
        planes_only = tc_out and E.planes_mode_ok()
        if planes_only:
            pl["stem"].bn_tile = 128          # 128-column tiles: the planes-only epilogue variant of the wider tiles runs out of registers (measured 1.7x slower)
        stem = pl["stem"](feat, ar.act("heads.stem", (B, feat.H, feat.W, pl["stem"].Cout), dev, lo=tc_out), f32_out=not planes_only)
        out = ar.act("heads.out", (B, feat.H, feat.W, pl["out_channels"]), dev)
        for n in pl["names"]:
            layer, cin_off, cout_off, n_pad = pl["outs"][n]
            layer(stem.slice(cin_off, self.bbox_head.head_features), out.slice(cout_off, n_pad))
        self._hook("heads", out)
        return out

    def _resnet_core(self, pl, images, ar) -> E.Act:
        """KM3DCore.forward for a ResNet backbone (KM3D_core.py:52-58): deconv_layers(backbone(image)[-1]).  The transposed convs read and
        (in planes mode) write fp16 planes only: each one's consumer is the next transposed conv or the head stem, all tensor-core convs."""
        rn, dc = pl["resnet"], pl["deconv"]
        B, dev = images.shape[0], images.device
        planes = E.planes_mode_ok()
        x = rn.run(images, ar, tag="bb", f32_outputs=[not planes] * len(rn.p.out_indices))[-1]
        if rn.out_lo_stale[-1]:
            E.split_lo(x)
        for i, layer in enumerate(dc):
            last = i == len(dc) - 1
            f32 = not planes or (last and pl["stem"].engine != "tc16")
            Ho, Wo = layer.out_hw(x.H, x.W)
            x = layer(x, ar.act(f"core.deconv{i}", (B, Ho, Wo, layer.Cout), dev, lo=True), f32_out=f32)
        return x

    def launch(self, images, P2):
        images, P2 = self._device_inputs((images, "image"), (P2, "P2"))
        _, _, H, W = images.shape
        return self.decode_maps(self.network(images), P2, H, W)

    def _check_head(self, off):
        missing = [k for k in self.REQUIRED if k not in off]
        if missing:
            raise Vd3dError(f"{type(self).__name__} head_dict lacks {missing}")

    def decode_maps(self, out: E.Act, P2: torch.Tensor, H: int, W: int):
        """The head's get_bboxes on the head maps `out` ([B, H/4, W/4, out_channels], the channel offsets of the plan); split from
        `launch` so that tests can feed the decode with the oracle's maps."""
        off = self.prepare()["offsets"]
        self._check_head(off)
        B, dev = out.B, out.t.device
        caps = self._peak_caps(out.H * out.W)
        dec = self._decoder((B, str(dev)) + caps,
                            lambda: E.DecodeNms(B, 128, dev, ws_bytes=getattr(_lib.load(), self.WORKSPACE)(B, *caps)))
        call(self.DECODE, out.ptr, B, out.H, out.W, self.num_classes, out.cs, *[off[k] for k in self.REQUIRED], P2.data_ptr(),
             float(self.test_cfg.get("score_thr", 0.1)), float(self.test_cfg.get("nms_iou_thr", 0.5)), self.topk,
             *self._decode_scalars(W, H, caps), dec.ws.data_ptr(), dec.cap, dec.scores.data_ptr(), dec.boxes.data_ptr(), dec.cls.data_ptr(),
             dec.anchor.data_ptr(), dec.count.data_ptr(), dec.ncand.data_ptr(), E._stream())
        return dec


@DETECTOR_DICT.register_module
class MonoFlex(_CenterNetBase):
    """R/detectors/KM3D.py:90-96 + MonoFlexHead.get_bboxes (R/heads/monoflex_head.py:114-179)."""
    REQUIRED = ("hm", "bbox2d", "hps", "rot", "dim", "reg", "depth", "depth_uncertainty", "corner_uncertainty")
    DECODE, WORKSPACE = "vd3d_monoflex_decode", "vd3d_monoflex_decode_workspace"

    def _peak_caps(self, n_cells):
        return (_peak_capacity(self.num_classes * n_cells),)

    def _decode_scalars(self, W, H, caps):
        return (float(self.uncertainty_range[0]), float(self.uncertainty_range[1]), float(W), float(H)) + caps


@DETECTOR_DICT.register_module
class KM3D(_CenterNetBase):
    """R/detectors/KM3D.py:16-88 + KM3DHead.get_bboxes/_decode (R/heads/km3d_head.py:155-314) + gen_position
    (R/utils/rtm3d_utils.py:314-455)."""
    REQUIRED = ("hm", "wh", "hps", "rot", "dim", "prob", "reg", "hm_hp", "hp_offset")
    DECODE, WORKSPACE = "vd3d_km3d_decode", "vd3d_km3d_decode_workspace"
    WITH_POSITION_LOSS = True

    def _check_head(self, off):
        super()._check_head(off)
        if self.bbox_head.head_dict["hps"] != 18 or self.bbox_head.head_dict["hm_hp"] != 9:
            raise Vd3dError("KM3D decode expects 9 keypoints (hps = 18, hm_hp = 9)")

    def _peak_caps(self, n_cells):
        return _peak_capacity(self.num_classes * n_cells), _peak_capacity(n_cells)

    def _decode_scalars(self, W, H, caps):
        return (float(W), float(H)) + caps

    @staticmethod
    def _result(scores, boxes, cls):
        # the reference's KM3D returns cls_indexes with shape [K, 1] (km3d_head.py:276 slices dets[mask, 40:41])
        return scores, boxes, cls.view(-1, 1)


def km3d_cfg(obj_types=("Car", "Pedestrian", "Cyclist")):
    """cfg.detector of R/config/KM3D_example:127-165 with the DLA-34 backbone of BASELINE.json configs[3]."""
    from ..synth import AttrDict
    obj_types = list(obj_types)
    det = AttrDict(obj_types=obj_types, name="KM3D")
    det.backbone = AttrDict(name="dlanet", depth=34, out_indices=(0, 1, 2, 3, 4, 5), pretrained=None)
    det.head = AttrDict(num_classes=len(obj_types), num_joints=9, max_objects=32,
                        layer_cfg=AttrDict(input_features=64, head_features=256,
                                           head_dict={"hm": len(obj_types), "wh": 2, "hps": 18, "rot": 8, "dim": 3, "prob": 1, "reg": 2,
                                                      "hm_hp": 9, "hp_offset": 2}),
                        loss_cfg=AttrDict(gamma=2.0, rampup_length=100, output_w=320),
                        test_cfg=AttrDict(score_thr=0.1))     # the shipped config uses 0.3; 0.1 keeps detections with the synthetic weights
    det.loss = det.head.loss_cfg
    return det


def monoflex_cfg(obj_types=("Car", "Pedestrian", "Cyclist"), name: str = "MonoFlex"):
    """cfg.detector of R/config/Monoflex_example:127-165."""
    from ..synth import AttrDict
    obj_types = list(obj_types)
    det = AttrDict(obj_types=obj_types, name=name)
    det.backbone = AttrDict(name="dlanet", depth=34, out_indices=(0, 1, 2, 3, 4, 5), pretrained=None)
    det.head = AttrDict(num_classes=len(obj_types), num_joints=9, max_objects=32,
                        layer_cfg=AttrDict(input_features=64, head_features=256,
                                           head_dict={"hm": len(obj_types), "bbox2d": 4, "hps": 20, "rot": 8, "dim": 3, "reg": 2, "depth": 1,
                                                      "depth_uncertainty": 1, "corner_uncertainty": 3}),
                        loss_cfg=AttrDict(gamma=2.0, output_w=320.0), test_cfg=AttrDict(score_thr=0.1))
    det.loss = det.head.loss_cfg
    return det


def km3d_example_cfg(obj_types=("Car", "Pedestrian", "Cyclist"), score_thr: float = 0.3):
    """cfg.detector of R/config/KM3D_example:127-165 as shipped, with pretrained=False: no backbone name (a ResNet-18 whose stage 3 feeds
    the transposed-conv up-sampling), 256 head input features, 64 head features."""
    from ..synth import AttrDict
    obj_types = list(obj_types)
    det = AttrDict(obj_types=obj_types, name="KM3D")
    det.backbone = AttrDict(depth=18, pretrained=False, frozen_stages=-1, num_stages=4, out_indices=(3,), norm_eval=False,
                            dilations=(1, 1, 1, 1))
    det.head = AttrDict(num_classes=len(obj_types), num_joints=9, max_objects=32,
                        layer_cfg=AttrDict(input_features=256, head_features=64,
                                           head_dict={"hm": len(obj_types), "wh": 2, "hps": 18, "rot": 8, "dim": 3, "prob": 1, "reg": 2,
                                                      "hm_hp": 9, "hp_offset": 2}),
                        loss_cfg=AttrDict(gamma=2.0, rampup_length=100, output_w=1280 // 4),
                        test_cfg=AttrDict(score_thr=score_thr))
    det.loss = det.head.loss_cfg
    return det


def monoflex_resnet_cfg(obj_types=("Car", "Pedestrian", "Cyclist")):
    """cfg.detector of R/config/Monoflex_example with its commented-out ResNet-18 backbone (name='resnet', depth=18, out_indices=(3,))
    and the 256 head input features the transposed-conv up-sampling produces."""
    from ..synth import AttrDict
    det = monoflex_cfg(obj_types)
    det.backbone = AttrDict(name="resnet", depth=18, out_indices=(3,), pretrained=False)
    det.head.layer_cfg.input_features = 256
    return det


def build_synthetic_monoflex(seed: int = 0, name: str = "MonoFlex", backbone: str = "dla34"):
    """Random-init (seeded, de-degenerated) MonoFlex / KM3D: returns (detector, state_dict, cfg).  backbone 'dla34': `km3d_cfg` /
    `monoflex_cfg`; 'resnet18': `km3d_example_cfg` (score_thr 0.1, as `km3d_cfg`, to keep detections with the synthetic weights) /
    `monoflex_resnet_cfg`."""
    if backbone == "resnet18":
        cfg = km3d_example_cfg(score_thr=0.1) if name == "KM3D" else monoflex_resnet_cfg()
    elif backbone == "dla34":
        cfg = km3d_cfg() if name == "KM3D" else monoflex_cfg(name=name)
    else:
        raise ValueError(f"backbone must be 'dla34' or 'resnet18', got {backbone!r}")
    det = DETECTOR_DICT[name](cfg)
    sd = synth_load(det, seed)
    return det, sd, cfg
