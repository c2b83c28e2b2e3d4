"""`MonoFlex` / `KM3D` — DLA-34 + DCNv2 up-sampling + CenterNet-style heads on the GPU
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


def _peak_capacity(n_cells: int) -> int:
    """Capacity of a heat-map peak list: a 3x3 local maximum rules out its 8 neighbours, so a map of n cells has at most ~n / 4 peaks;
    power of two in [1024, 8192] (the library's limit: more peaks than that are reported as an overflow, never truncated).  The decode
    kernels sort only the occupied part of a list, so a generous capacity costs memory, not time."""
    cap = 1024
    while cap < min(8192, (n_cells + 3) // 4):
        cap <<= 1
    return cap


class KM3DCoreP(M.Holder):
    """keys of KM3DCore (R/detectors/KM3D_core.py:10-50) for the DLA backbone."""

    def __init__(self, backbone_arguments):
        super().__init__()
        args = dict(backbone_arguments)
        name = str(args.get("name", "dlanet")).lower()
        if name not in ("dla", "dlanet"):
            raise NotImplementedError("KM3DCore on the B200 path supports the DLA backbone (the shipped KM3D / MonoFlex configs)")
        self.backbone = DLAP(**args)
        self.deconv_layers = DLASegUpsampleP(input_channels=[16, 32, 64, 128, 256, 512], down_ratio=4, final_kernel=1, last_level=5, out_channel=64)
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
        pl = dict(dla=DLARunner(self.core.backbone, dev, first_used_level=self.core.deconv_layers.first_level), up=DLAUpRunner(self.core.deconv_layers, dev))
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
            raise Vd3dError(f"{type(self).__name__}: image size {H}x{W} must be a multiple of 32 (DLA-34 has 5 stride-2 levels)")
        ys = pl["dla"].run(images, ar)
        feat = pl["up"].run(ys, ar)                       # [B, H/4, W/4, 64]
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


def build_synthetic_monoflex(seed: int = 0, name: str = "MonoFlex"):
    """Random-init (seeded, de-degenerated) MonoFlex / KM3D: returns (detector, state_dict, cfg)."""
    cfg = km3d_cfg() if name == "KM3D" else monoflex_cfg(name=name)
    det = DETECTOR_DICT[name](cfg)
    sd = synth_load(det, seed)
    return det, sd, cfg
