"""`RetinaNet` — the 2-D detector of R/detectors/retinanet_2d.py:75-151 (config R/config/RetinaNet_example) on the GPU.

Protocol (R/pipelines/testers.py): ``module([image[1,3,H,W], P2])`` -> ``(scores[K] f32, bboxes[K,4] f32, labels[K] int64)``; a 3-element
list means training (raises: out of scope).  ``forward_batch(images)`` is the batched entry point, ``launch(images, P2)`` the
stream-ordered one (graphs.GraphedStep, pipeline.StreamedInference).

  ResNet (out_indices (1, 2, 3): C3 / C4 / C5)
  -> FPN: lateral 1x1 convs, the top-down `lat[i-1] += nearest_up2(lat[i])` fused into the lateral conv's residual read
     (ConvLayer(res_up=True)), 3x3 fpn convs, P6 = 3x3/2 on C5, P7 = 3x3/2 on P6, no ReLU
  -> head: the same cls / reg towers (stacked 3x3 conv + ReLU) and output convs on every level, each layer one persistent launch over all
     levels and the whole batch (ConvLayer.run_levels); the cls output conv is padded to a multiple of 16 zero-weight columns so that it
     runs on the tensor cores (the decode reads it with that channel pitch)
  -> device decode (vd3d_retina_decode): max-sigmoid score, top-k, _decode, class-agnostic NMS, post-NMS score threshold.
"""
from __future__ import annotations

import ctypes
from typing import List

import numpy as np
import torch
import torch.nn as nn

from .. import engine as E
from .. import _lib
from .._lib import Vd3dError, call
from ..anchors import grid_anchors
from ..plugin import DETECTOR_DICT
from . import modules as M
from .base import NativeDetector, synth_load
from .stereo3d import ResNetRunner


class RetinaDecode(E.DecodeNms):
    """Fixed-capacity outputs of the RetinaNet decode for a batch: the DecodeNms buffers (boxes [B, cap, 11] with columns 4..10 zero, so
    the record block of parallel.pack_records_device carries the 4 box columns) plus the top-k workspace."""

    def __init__(self, B: int, N: int, cap: int, device):
        super().__init__(B, cap, device, ws_bytes=_lib.load().vd3d_retina_decode_workspace(B, N, cap))
        self.N = N

    def run_levels(self, cls_levels, reg_levels, level_pix, cls_cs, reg_cs, anchors, A, ncls, nms_pre, means, stds, score_thr, iou_thr):
        L = len(level_pix)
        cls_arr = (ctypes.c_void_p * L)(*[t.data_ptr() for t in cls_levels])
        reg_arr = (ctypes.c_void_p * L)(*[t.data_ptr() for t in reg_levels])
        pix_arr = (ctypes.c_int * L)(*[int(v) for v in level_pix])
        m4 = (ctypes.c_float * 4)(*[float(v) for v in means])
        s4 = (ctypes.c_float * 4)(*[float(v) for v in stds])
        call("vd3d_retina_decode", L, cls_arr, reg_arr, pix_arr, int(cls_cs), int(reg_cs), anchors.data_ptr(), self.B, self.N, int(A), int(ncls),
             int(nms_pre), m4, s4, float(np.float32(score_thr)), float(iou_thr), self.cap, self.ws.data_ptr(),
             self.scores.data_ptr(), self.boxes.data_ptr(), self.cls.data_ptr(), self.anchor.data_ptr(), self.count.data_ptr(),
             self.ncand.data_ptr(), E._stream())

    def post_opt(self, *a, **k):
        raise Vd3dError("RetinaNet is a 2-D detector: there is no 3-D yaw to refine")

    def post_forward(self, *a, **k):
        raise Vd3dError("RetinaNet is a 2-D detector: the 3-D post-forward geometry (geometry=True) does not apply")


def _cfg_get(d, k, default):
    """test_cfg lookup the way the reference does it (`getattr(test_cfg, k, default)` on an EasyDict; a plain dict also works)"""
    try:
        return d[k]
    except (KeyError, TypeError):
        return getattr(d, k, default)


@DETECTOR_DICT.register_module
class RetinaNet(NativeDetector):
    """R/detectors/retinanet_2d.py:75-151 (inference).  `network_cfg` is the reference's `cfg.detector` (backbone, neck, head)."""

    def __init__(self, network_cfg):
        super().__init__()
        self.obj_types = network_cfg["obj_types"]
        bb, neck, head = dict(network_cfg["backbone"]), dict(network_cfg["neck"]), dict(network_cfg["head"])
        in_ch, num_outs = list(neck["in_channels"]), int(neck["num_outs"])
        if num_outs < len(in_ch):
            raise ValueError(f"neck.num_outs = {num_outs} < len(in_channels) = {len(in_ch)} is not supported (the reference's FPN drops no level)")
        out_idx = tuple(bb.get("out_indices", (-1, 0, 1, 2, 3)))
        if len(out_idx) != len(in_ch) or -1 in out_idx or list(out_idx) != sorted(out_idx):
            raise ValueError(f"backbone.out_indices {out_idx} must name one ascending ResNet stage per FPN input ({len(in_ch)})")
        acfg = head["anchors_cfg"]
        self.anchors_cfg = {k: acfg[k] for k in ("pyramid_levels", "strides", "sizes", "ratios", "scales")}
        if len(self.anchors_cfg["pyramid_levels"]) != num_outs:
            raise ValueError(f"anchors_cfg.pyramid_levels has {len(self.anchors_cfg['pyramid_levels'])} levels, the FPN {num_outs} outputs")
        self.num_anchors = len(acfg["ratios"]) * len(acfg["scales"])
        self.num_classes = int(head.get("num_classes", 3))
        self.reg_output = int(head.get("reg_output", 4))
        if self.reg_output != 4:
            raise ValueError("head.reg_output must be 4 (the (dx, dy, dw, dh) layout of RetinanetHead._decode)")
        self.target_means = [float(v) for v in head.get("target_means", [0.0] * 4)]
        self.target_stds = [float(v) for v in head.get("target_stds", [1.0] * 4)]
        self.test_cfg = head.get("test_cfg", {}) or {}
        self.nms_pre = int(_cfg_get(self.test_cfg, "nms_pre", 1000))
        self.score_thr = float(_cfg_get(self.test_cfg, "score_thr", 0.5))
        self.nms_iou_thr = float(_cfg_get(self.test_cfg, "nms_iou_thr", 0.5))
        # `cls_agnositc` (sic, retinanet_head.py:285) is never set by a config, so the reference always runs class-agnostic NMS
        if not bool(_cfg_get(self.test_cfg, "cls_agnositc", True)):
            raise ValueError("test_cfg.cls_agnositc=False: the reference's class-aware NMS branch cannot run (unsqueeze() without a dim)")
        if self.nms_pre > 4096:
            raise ValueError(f"test_cfg.nms_pre = {self.nms_pre} exceeds the NMS capacity (4096 candidates per image)")
        self.network_cfg = network_cfg
        self.core = M.RetinaNetCoreP(bb, neck)
        for i, s in enumerate(out_idx):
            if self.core.backbone.out_channels(s) != in_ch[i]:
                raise ValueError(f"neck.in_channels[{i}] = {in_ch[i]} but ResNet stage {s} has {self.core.backbone.out_channels(s)} channels")
        self.bbox_head = M.RetinaHeadP(self.num_anchors, int(head.get("stacked_convs", 4)), int(head.get("in_channels", 256)),
                                       int(head.get("feat_channels", 256)), self.num_classes, self.reg_output, dict(head.get("loss_cfg", {}) or {}))
        self._anchors = {}

    # ---- plan (packed weights) -------------------------------------------------------------------------------
    def build_plan(self, dev) -> dict:
        neck, hd = self.core.neck, self.bbox_head
        conv = lambda c, **kw: E.ConvLayer(c.weight, c.bias, None, device=dev, **kw)
        n_in = len(neck.in_channels)
        pl = dict(backbone=ResNetRunner(self.core.backbone, dev),
                  lateral=[conv(c) for c in neck.lateral_convs],
                  fpn=[conv(c, pad=1, stride=1 if i < n_in else 2) for i, c in enumerate(neck.fpn_convs)],
                  cls=[conv(m.sequence[0], pad=1, relu=True) for m in hd.cls_conv],
                  reg=[conv(m.sequence[0], pad=1, relu=True) for m in hd.reg_conv],
                  reg_out=conv(hd.retina_reg[0], pad=1))
        # cls output: padded to a multiple of 16 zero-weight columns (27 -> 32 at A = 9, C = 3) so that it runs on the tensor cores
        c = hd.retina_cls[0]
        n = c.out_channels
        npad = (n + 15) // 16 * 16
        w = torch.zeros(npad, *c.weight.shape[1:], dtype=torch.float64)
        b = torch.zeros(npad, dtype=torch.float64)
        w[:n], b[:n] = c.weight.detach().cpu().double(), c.bias.detach().cpu().double()
        pl["cls_out"] = E.ConvLayer(w, b, None, pad=1, device=dev)
        for l in pl["lateral"] + pl["fpn"] + pl["cls"] + pl["reg"] + [pl["reg_out"], pl["cls_out"]]:
            if l.engine != "tc16":
                raise Vd3dError(f"RetinaNet runs on the fp16-split tensor-core engine (VD3D_CONV_ENGINE=tc16); a {l.Cin}->{l.Cout} conv got '{l.engine}'")
        return pl

    def _anchor_table(self, H, W, dev) -> torch.Tensor:
        key = (H, W, str(dev))
        if key not in self._anchors:
            a = self.anchors_cfg
            a64 = grid_anchors((H, W), a["pyramid_levels"], a["strides"], a["sizes"], a["ratios"], a["scales"])
            self._anchors[key] = torch.tensor(a64.astype(np.float32)).to(dev).contiguous()
        return self._anchors[key]

    # ---- forward -------------------------------------------------------------------------------------------------
    def features(self, images: torch.Tensor) -> List[E.Act]:
        """backbone + FPN: the pyramid levels P3 .. P7 (fp32 with fresh fp16 planes)."""
        return self.fpn(self.backbone(images))

    def backbone(self, images: torch.Tensor) -> List[E.Act]:
        """ResNet C3 / C4 / C5 with fresh fp16 planes."""
        pl = self.prepare()
        feats = pl["backbone"].run(images, self._arena, tag="bb")
        for f, stale in zip(feats, pl["backbone"].out_lo_stale):
            if stale:
                E.split_lo(f)
        return feats

    def fpn(self, feats: List[E.Act]) -> List[E.Act]:
        pl = self.prepare()
        ar = self._arena
        B, dev = feats[0].B, feats[0].t.device
        # laterals from the top: lat[i] = conv1x1(C_i) + nearest_up2(lat[i + 1]), the add fused into the conv epilogue
        lat = [None] * len(feats)
        for i in range(len(feats) - 1, -1, -1):
            f, layer = feats[i], pl["lateral"][i]
            out = ar.act(f"fpn.lat{i}", (B, f.H, f.W, layer.Cout), dev, lo=True)
            lat[i] = layer(f, out) if i == len(feats) - 1 else layer(f, out, res=lat[i + 1], res_up=True)
        outs = []
        for i, layer in enumerate(pl["fpn"]):
            src = lat[i] if i < len(feats) else (feats[-1] if i == len(feats) else outs[-1])
            Ho, Wo = layer.out_hw(src.H, src.W)
            outs.append(layer(src, ar.act(f"fpn.P{i}", (B, Ho, Wo, layer.Cout), dev, lo=True)))
        return outs

    def head(self, levels: List[E.Act]):
        """The shared-weight towers and output convs: every layer is ONE launch over all levels and the whole batch (`ConvLayer.run_levels`,
        the levels' activations concatenated in one buffer per layer).  Returns per level (cls [B, h, w, pitch], reg [B, h, w, A * 4])."""
        pl = self.prepare()
        ar = self._arena
        B, dev = levels[0].B, levels[0].t.device
        hws = [(x.H, x.W) for x in levels]
        out = {}
        for br, tower, last in (("cls", pl["cls"], pl["cls_out"]), ("reg", pl["reg"], pl["reg_out"])):
            a = list(levels)
            for j, layer in enumerate(tower):
                a = layer.run_levels(a, ar.level_acts(f"head.{br}{j % 2}", B, hws, layer.Cout, dev, lo=True))
            out[br] = last.run_levels(a, ar.level_acts(f"head.{br}.out", B, hws, last.Cout, dev))
        return list(zip(out["cls"], out["reg"]))

    def launch(self, images, P2=None):
        [images] = self._device_inputs((images, "image"))
        B, _, H, W = images.shape
        if H % 32 or W % 32:
            raise Vd3dError(f"RetinaNet: image size {H}x{W} must be a multiple of 32 (the FPN top-down add needs every level twice the next)")
        levels = self.features(images)
        for i, p in enumerate(levels):
            self._hook(f"P{i}", p)
        heads = self.head(levels)
        for i, (c, r) in enumerate(heads):
            self._hook(f"cls{i}", c), self._hook(f"reg{i}", r)
        return self.decode(heads, H, W)

    def decode(self, heads, H: int, W: int) -> RetinaDecode:
        dev = heads[0][0].t.device
        B = heads[0][0].B
        anchors = self._anchor_table(H, W, dev)
        N = anchors.shape[0]
        pix = [c.H * c.W for c, _ in heads]
        if sum(pix) * self.num_anchors != N:
            raise Vd3dError(f"RetinaNet: the head levels hold {sum(pix) * self.num_anchors} anchors, the anchor table {N}")
        cap = self.nms_pre if 0 < self.nms_pre < N else N
        if cap > 4096:
            raise Vd3dError(f"RetinaNet: {cap} NMS candidates per image exceed the capacity (4096): set test_cfg.nms_pre <= 4096")
        dec = self._decoder((B, N, cap, str(dev)), lambda: RetinaDecode(B, N, cap, dev))
        dec.run_levels([c.t for c, _ in heads], [r.t for _, r in heads], pix, heads[0][0].cs, heads[0][1].cs, anchors, self.num_anchors,
                       self.num_classes, self.nms_pre, self.target_means, self.target_stds, self.score_thr, self.nms_iou_thr)
        return dec

    @staticmethod
    def _result(scores, boxes, cls):
        return scores, boxes[:, :4], cls          # the 2-D box columns of the DecodeNms rows


def build_synthetic_retinanet(seed: int = 0, depth: int = 50, nms_pre: int = 1000):
    """Random-init (seeded) RetinaNet of the example config: returns (detector, state_dict, cfg)."""
    from .. import synth
    cfg = synth.retinanet_cfg(depth=depth, nms_pre=nms_pre)
    det = DETECTOR_DICT["RetinaNet"](cfg)
    sd = synth_load(det, seed)
    return det, sd, cfg
