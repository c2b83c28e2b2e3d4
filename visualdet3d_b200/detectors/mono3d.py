"""`Yolo3D` and `GroundAwareYolo3D` — monocular anchor-based 3-D detectors on the GPU
(drop-ins for R/detectors/yolomono3d_detector.py:55-138; cores R/detectors/yolomono3d_core.py:9-18).

Protocol (R/pipelines/testers.py:24-25): ``module([image[1,3,H,W], P2[1,3,4]])`` -> ``(scores[K], bboxes[K,11], cls[K])``;
a 3-element list means training (raises: out of scope).  ``forward_batch(images, P2)`` is the batched entry point.

  Yolo3D            : ResNet(out_indices=(2,)) -> cls tower | reg tower = DCNv2 + BN + ReLU, conv + BN + ReLU, conv
                      (R/heads/detection_3d_head.py:47-88)
  GroundAwareYolo3D : same backbone -> cls tower | reg tower = LookGround (Ground-Aware Convolution), conv+BN+ReLU x2, conv
                      (yolomono3d_detector.py:12-53, R/lib/look_ground.py)
"""
from __future__ import annotations

from typing import Optional

import torch

from .. import engine as E
from .._lib import Vd3dError, call
from ..plugin import DETECTOR_DICT
from . import modules as M
from .base import Anchor3DDetector, synth_load
from .stereo3d import ResNetRunner, cls_tower_runner, run_cls_tower


class LookGroundRunner:
    """LookGround.forward (R/lib/look_ground.py:24-71): disp conv (conv engine, Cout padded to 16) -> sampling kernel ->
    1x1 `extract` conv with alpha folded into its weights, residual x and ReLU fused into the conv epilogue."""

    def __init__(self, p: M.LookGroundP, device):
        C = p.extract.out_channels
        self.C, self.baseline, self.elev = C, float(p.baseline), float(p.relative_elevation)
        dw = torch.zeros(16, C, 3, 3)
        dw[0] = p.disp_create[0].weight.detach().cpu()[0]
        db = torch.zeros(16)
        db[0] = p.disp_create[0].bias.detach().cpu()[0]
        self.disp = E.ConvLayer(dw, db, None, pad=1, relu=False, device=device)
        alpha = float(p.alpha.detach().cpu()[0])
        w = p.extract.weight.detach().cpu().double()[:, :, 0, 0]          # [C, 1 + C]: input channel 0 = disparity plane
        self.cin_pad = C + 32
        wp = torch.zeros(C, self.cin_pad, 1, 1, dtype=torch.float64)
        wp[:, :C, 0, 0] = w[:, 1:] * alpha
        wp[:, C, 0, 0] = w[:, 0] * alpha
        self.extract = E.ConvLayer(wp, p.extract.bias.detach().cpu().double() * alpha, None, relu=True, device=device)

    def run(self, x: E.Act, P2: torch.Tensor, arena: E.Arena, tag: str = "gac") -> E.Act:
        """x: stride-16 features with a fresh lo companion (if the convs are tensor-core).  Returns relu(x + extract(sampled) * alpha)."""
        B, H, W, dev = x.B, x.H, x.W, x.t.device
        d = self.disp(x, arena.act(tag + ".disp", (B, H, W, 16), dev))
        S = arena.act(tag + ".S", (B, H, W, self.cin_pad), dev, lo=self.extract.engine != "simt", zero=True)
        call("vd3d_look_ground_sample", x.ptr, B, H, W, x.C, x.cs, x.co, d.ptr, d.cs, 0, P2.data_ptr(), self.baseline, self.elev,
             S.ptr, S.lo_ptr, S.cs, E._stream())
        if S.h16:
            E.split_lo(S)
        return self.extract(S, arena.act(tag + ".out", (B, H, W, self.C), dev, lo=True), res=x)


class _Mono3DBase(Anchor3DDetector):
    head_cls = None

    def __init__(self, network_cfg):
        super().__init__(network_cfg)
        self.bbox_head = self.head_cls(**self.head_kwargs)
        self.core = M.YoloMono3DCoreP(dict(network_cfg["backbone"]))

    def reg_plan(self, dev) -> dict:  # pragma: no cover
        raise NotImplementedError

    def build_plan(self, dev) -> dict:
        pl = dict(backbone=ResNetRunner(self.core.backbone, dev), cls=cls_tower_runner(self.bbox_head.cls_feature_extraction, dev))
        pl.update(self.reg_plan(dev))
        return pl

    def run_reg(self, pl, feat: E.Act, P2, arena, tower: bool = True) -> E.Act:  # pragma: no cover
        """the reg tower up to the input of its output conv pl["reg_out"]; tower=False: up to the input of `reg_tower(pl)`"""
        raise NotImplementedError

    def launch(self, images, P2):
        images, P2 = self._device_inputs((images, "image"), (P2, "P2"))
        B, _, H, W = images.shape
        if H % 16 or W % 16:
            raise Vd3dError(f"{type(self).__name__}: image size {H}x{W} must be a multiple of 16")
        pl = self.prepare()
        ar = self._arena
        feat = pl["backbone"].run(images, ar)[0]               # YoloMono3DCore.forward: x = backbone(image)[0]
        if pl["backbone"].last_lo_stale:
            E.split_lo(feat)
        self._hook("features", feat)
        cls = run_cls_tower(pl["cls"], feat, ar)
        sparse = self.sparse_reg(pl["reg_out"], B, feat.H, feat.W)
        tower = self.tiled_tower(pl, sparse, feat.H, feat.W)
        x = self.run_reg(pl, feat, P2, ar, tower=not tower)
        if sparse:
            return self.decode(cls, x, P2, H, W, reg_out=pl["reg_out"], tower=tower)
        reg = self.run_reg_out(pl["reg_out"], x)
        self._hook("cls_preds", cls), self._hook("reg_preds", reg)
        return self.decode(cls, reg, P2, H, W)


@DETECTOR_DICT.register_module
class Yolo3D(_Mono3DBase):
    """R/detectors/yolomono3d_detector.py:55-129."""
    head_cls = M.MonoHeadP

    def reg_plan(self, dev):
        rt = self.bbox_head.reg_feature_extraction
        d = rt[0]
        return dict(
            dcn=E.DeformConvLayer(d.weight, d.bias, d.conv_offset.weight, d.conv_offset.bias, E.bn_dict(rt[1]), d.stride, d.padding,
                                  d.dilation, d.deformable_groups, relu=True, device=dev),
            reg1=E.ConvLayer(rt[3].weight, rt[3].bias, E.bn_dict(rt[4]), pad=1, relu=True, device=dev),
            reg_out=E.ConvLayer(rt[6].weight, rt[6].bias, None, pad=1, relu=False, device=dev))

    def run_reg(self, pl, feat, P2, ar, tower=True):
        B, h, w, dev = feat.B, feat.H, feat.W, feat.t.device
        tc = lambda l: l.engine != "simt"
        a = pl["dcn"](feat, ar.act("R1", (B, h, w, pl["dcn"].Cout), dev, lo=True), ar, "dcn")
        if tc(pl["reg1"]) and not tc(pl["dcn"].main):
            E.split_lo(a)
        a = pl["reg1"](a, ar.act("R2", (B, h, w, pl["reg1"].Cout), dev, lo=True))
        if tc(pl["reg_out"]) and not tc(pl["reg1"]):
            E.split_lo(a)
        return a


@DETECTOR_DICT.register_module
class GroundAwareYolo3D(_Mono3DBase):
    """R/detectors/yolomono3d_detector.py:131-138 (GroundAwareHead :12-53)."""
    head_cls = M.GroundAwareHeadP

    def reg_plan(self, dev):
        rt = self.bbox_head.reg_feature_extraction
        return dict(gac=LookGroundRunner(rt[0], dev),
                    reg0=E.ConvLayer(rt[1].weight, rt[1].bias, E.bn_dict(rt[2]), pad=1, relu=True, device=dev),
                    reg1=E.ConvLayer(rt[4].weight, rt[4].bias, E.bn_dict(rt[5]), pad=1, relu=True, device=dev),
                    reg_out=E.ConvLayer(rt[7].weight, rt[7].bias, None, pad=1, relu=False, device=dev))

    def reg_tower(self, pl):
        return [(pl["reg0"], "R1", None), (pl["reg1"], "R2", None)]

    def run_reg(self, pl, feat, P2, ar, tower=True):
        B, h, w, dev = feat.B, feat.H, feat.W, feat.t.device
        tc = lambda l: l.engine != "simt"
        a = pl["gac"].run(feat, P2, ar)
        self._hook("gac", a)
        if tc(pl["reg0"]) and not tc(pl["gac"].extract):
            E.split_lo(a)
        if not tower:
            return a
        for k, name in (("reg0", "R1"), ("reg1", "R2")):
            nxt = pl["reg1"] if k == "reg0" else pl["reg_out"]
            a = pl[k](a, ar.act(name, (B, h, w, pl[k].Cout), dev, lo=True))
            if tc(nxt) and not tc(pl[k]):
                E.split_lo(a)
        return a


def build_synthetic_mono3d(kind: str = "Yolo3D", seed: int = 0, depth: Optional[int] = None, workdir: Optional[str] = None):
    """Random-init (seeded, de-degenerated) mono detector + priors: returns (detector, state_dict, cfg, (prior_mean, prior_std))."""
    import tempfile
    from .. import synth
    obj_types = ["Car"]
    pm, ps = synth.synth_priors(16, 2, obj_types)
    d = workdir or tempfile.mkdtemp(prefix="vd3d_priors_")
    synth.write_priors(d, pm, ps, obj_types)
    cfg = synth.mono3d_cfg(d, kind, obj_types, depth)
    det = DETECTOR_DICT[kind](cfg)
    sd = synth_load(det, seed)
    return det, sd, cfg, (pm, ps)
