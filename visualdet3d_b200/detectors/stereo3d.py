"""`Stereo3D` — YOLOStereo3D inference forward on the GPU (drop-in for R/detectors/yolostereo3d_detector.py:16-103).

Same construction (`DETECTOR_DICT['Stereo3D'](cfg.detector)`), same checkpoint keys, same list protocol:
``module([left[1,3,H,W], right, P2[1,3,4], P3])`` -> ``(scores[K], bboxes[K,11], cls_indexes[K] int64)``.
New: ``forward_batch`` runs B pairs at once (the reference asserts B == 1, :78) and returns one triple per image.

Execution plan per forward (all kernels from libvd3d_b200, NHWC fp32, every torch.cat fused into producers):
  NCHW->NHWC(4ch) -> stem 7x7s2 -> maxpool -> ResNet stages (conv+BN+ReLU+residual fused)
  -> PSMCosine x2 (written straight into the ghost-module concat buffers) + concat-volume/Conv3d x2
  -> CostVolumePyramid -> features[1408] -> cls / reg towers -> anchors mask -> decode + NMS.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import numpy as np
import torch
import torch.nn as nn

from .. import engine as E
from .._lib import Vd3dError, call
from ..plugin import DETECTOR_DICT
from . import modules as M
from .base import Anchor3DDetector, synth_load


class ResNetRunner:
    """Folded ResNet stages (R/backbones/resnet.py:184-198) over the engine."""

    def __init__(self, p: M.ResNetP, device):
        self.p = p
        self.stem = E.ConvLayer(p.conv1.weight, None, E.bn_dict(p.bn1), stride=2, pad=3, relu=True, device=device, cin_pad=4)
        # tensor-core stem (default with the fp16-split engine): image -> fp16 row planes -> KHx1 conv over 64 virtual channels
        import os
        self.stem_tc = None
        if E.conv_engine_default() == "tc16" and os.environ.get("VD3D_STEM_TC", "1") != "0" and str(device).startswith("cuda"):
            self.stem_tc = E.StemLayer(p.conv1.weight, E.bn_dict(p.bn1), stride=2, pad=3, relu=True, device=device)
        self.stages = []
        for i in range(p.num_stages):
            blocks = []
            for blk in getattr(p, f"layer{i + 1}"):
                d = {}
                if isinstance(blk, M.BasicBlockP):
                    d["kind"] = "basic"
                    d["c1"] = E.ConvLayer(blk.conv1.weight, None, E.bn_dict(blk.bn1), stride=blk.stride, pad=1, relu=True, device=device)
                    d["c2"] = E.ConvLayer(blk.conv2.weight, None, E.bn_dict(blk.bn2), stride=1, pad=blk.dilation, dil=blk.dilation, relu=True, device=device)
                else:
                    d["kind"] = "bottle"
                    d["c1"] = E.ConvLayer(blk.conv1.weight, None, E.bn_dict(blk.bn1), relu=True, device=device)
                    d["c2"] = E.ConvLayer(blk.conv2.weight, None, E.bn_dict(blk.bn2), stride=blk.stride, pad=blk.dilation, dil=blk.dilation, relu=True, device=device)
                    d["c3"] = E.ConvLayer(blk.conv3.weight, None, E.bn_dict(blk.bn3), relu=True, device=device)
                if blk.downsample is not None:
                    d["ds"] = E.ConvLayer(blk.downsample[0].weight, None, E.bn_dict(blk.downsample[1]), stride=blk.stride, relu=False, device=device)
                blocks.append(d)
            self.stages.append(blocks)

    def run(self, img_nchw, arena: E.Arena, tag: str = "bb", on_output=None, f32_outputs=None) -> List[E.Act]:
        """`img_nchw`: [B, 3, H, W], or a list of such tensors forming the batch in order (stereo: [left, right]; the parts are read in
        place, the reference's `torch.cat([left, right])` copy does not exist).
        Inside the stages every activation lives as fp16 (hi, lo) planes only (`engine.planes_mode_ok`): a block's convs, its residual and
        the tensor-core PSMCosine read planes, so no fp32 copy is written or re-read (half the activation traffic of the 64 / 128-channel
        layers).  `f32_outputs[j]` says whether returned feature map j also needs its fp32 tensor (default: yes).
        on_output(act, lo_stale) -> lo_stale: called as soon as a returned feature map exists, i.e. while it is still
        L2-resident (the stereo plan launches the cost-volume kernel of that scale from it)."""
        parts = list(img_nchw) if isinstance(img_nchw, (list, tuple)) else [img_nchw]
        dev = parts[0].device
        _, _, H, W = parts[0].shape
        B = sum(int(p.shape[0]) for p in parts)
        Hs, Ws = self.stem.out_hw(H, W)
        Hp, Wp = (Hs + 2 - 3) // 2 + 1, (Ws + 2 - 3) // 2 + 1
        import os
        fuse_pool = self.stem_tc is not None and -1 not in self.p.out_indices and os.environ.get("VD3D_STEM_POOL", "1") != "0"
        x = None
        if fuse_pool:
            # stem conv + BN + ReLU + max-pool in ONE kernel (the 64-channel half-resolution stem output never reaches HBM)
            # (row-strip kernel: the pooled tensor is written as the fp16 planes layer 1 reads; its fp32 copy only when planes mode is off)
            pooled = self.stem_tc(parts, arena.act(tag + ".pool", (B, Hp, Wp, 64), dev, lo=True), arena, tag, pool=True, f32_out=not E.planes_mode_ok())
        elif self.stem_tc is not None:
            x = self.stem_tc(parts, arena.act(tag + ".stem", (B, Hs, Ws, 64), dev), arena, tag)
        else:
            x0 = arena.act(tag + ".in4", (B, H, W, 4), dev, zero=True)
            b0 = 0
            for p in parts:
                E.nchw_to_nhwc(p, x0.batch(b0, b0 + int(p.shape[0])))
                b0 += int(p.shape[0])
            x = self.stem(x0, arena.act(tag + ".stem", (B, Hs, Ws, 64), dev))
        outs = []
        self.out_lo_stale = []             # per returned feature map: True if its tensor-core companion is not up to date
        if -1 in self.p.out_indices:
            outs.append(x)
            self.out_lo_stale.append(True)
        x = pooled if fuse_pool else E.maxpool3x3s2(x, arena.act(tag + ".pool", (B, Hp, Wp, 64), dev, lo=True))
        fresh = not (fuse_pool and getattr(self.stem_tc, "wrote_planes", False))     # True: x.lo is stale (x was written by a kernel that does not write the planes)
        plm = E.planes_mode_ok()
        n_ret = len(outs)                  # index of the next returned feature map

        def want_f32(stage_idx, last_block, out_layer):
            """fp32 copy of a block output: needed only if it is a returned map whose consumers read fp32 (or planes mode is off)"""
            if not E.planes_only_ok(out_layer):
                return True
            if last_block and stage_idx in self.p.out_indices:
                return True if f32_outputs is None else bool(f32_outputs[n_ret])
            return False

        def feed(layer, a, stale):
            """make sure `a` carries a valid lo companion if `layer` runs on the tensor cores"""
            if layer.engine != "simt" and stale:
                E.split_lo(a)
                return False
            return stale

        for i, blocks in enumerate(self.stages):
            for j, d in enumerate(blocks):
                name = f"{tag}.s{i}b{j}"
                if d["kind"] == "basic":
                    c1, c2 = d["c1"], d["c2"]
                    Ho, Wo = c1.out_hw(x.H, x.W)
                    fresh = feed(c1, x, fresh)
                    t = c1(x, arena.act(name + ".t", (B, Ho, Wo, c1.Cout), dev, lo=True), f32_out=not (E.planes_only_ok(c1) and c2.engine == "tc16"))
                    feed(c2, t, c1.engine == "simt")
                    r = x if "ds" not in d else d["ds"](x, arena.act(name + ".r", (B, Ho, Wo, c2.Cout), dev))
                    x = c2(t, arena.act(name + ".o", (B, Ho, Wo, c2.Cout), dev, lo=True), res=r, f32_out=want_f32(i, j == len(blocks) - 1, c2))
                    fresh = c2.engine == "simt"
                else:
                    c1, c2, c3 = d["c1"], d["c2"], d["c3"]
                    fresh = feed(c1, x, fresh)
                    t1 = c1(x, arena.act(name + ".t1", (B, x.H, x.W, c1.Cout), dev, lo=True), f32_out=not (E.planes_only_ok(c1) and c2.engine == "tc16"))
                    Ho, Wo = c2.out_hw(x.H, x.W)
                    feed(c2, t1, c1.engine == "simt")
                    t2 = c2(t1, arena.act(name + ".t2", (B, Ho, Wo, c2.Cout), dev, lo=True), f32_out=not (E.planes_only_ok(c2) and c3.engine == "tc16"))
                    feed(c3, t2, c2.engine == "simt")
                    if "ds" in d:
                        fresh = feed(d["ds"], x, fresh)
                        r = d["ds"](x, arena.act(name + ".r", (B, Ho, Wo, c3.Cout), dev))
                    else:
                        r = x
                    x = c3(t2, arena.act(name + ".o", (B, Ho, Wo, c3.Cout), dev, lo=True), res=r, f32_out=want_f32(i, j == len(blocks) - 1, c3))
                    fresh = c3.engine == "simt"
            if i in self.p.out_indices:
                outs.append(x)
                n_ret += 1
                if on_output is not None:
                    fresh = on_output(x, fresh)
                self.out_lo_stale.append(fresh)
        self.last_lo_stale = fresh
        return outs


class GhostRunner:
    """ResGhostModule (R/lib/ghost_module.py:46-64): out = cat[x, x1, x2][:, :oup], executed in place in the concat buffer:
    x already sits in channels [0, inp) of `buf`; x1 -> [inp, inp+init), x2 -> [inp+init, ...)."""

    def __init__(self, p: M.GhostP, device):
        self.p = p
        k = p.kernel_size
        self.primary = E.ConvLayer(p.primary_conv[1].weight, None, E.bn_dict(p.primary_conv[2]), pad=k // 2, relu=True, device=device)
        self.cheap = E.DwConvLayer(p.cheap_operation[0].weight, E.bn_dict(p.cheap_operation[1]), relu=True, device=device)
        assert p.new_channels == p.init_channels, "depthwise multiplier != 1 is not on the path"
        assert p.inp + p.init_channels + p.new_channels == p.oup, "channel truncation [:oup] is not on the path"

    def run(self, buf: E.Act):
        """`buf` channels [0, inp) hold x.  On return every channel of `buf` carries a valid lo companion if it has one."""
        p = self.p
        x = buf.slice(0, p.inp)
        if self.primary.engine != "simt":
            E.split_lo(x)
        x1 = self.primary(x, buf.slice(p.inp, p.init_channels))
        x2 = self.cheap(x1, buf.slice(p.inp + p.init_channels, p.new_channels))
        if buf.lo is not None:
            if self.primary.engine == "simt":
                E.split_lo(buf)
            else:
                E.split_lo(x2)
        return buf


def cls_tower_runner(ct, device):
    """conv3x3+ReLU, conv3x3+ReLU, conv3x3 (R/heads/detection_3d_head.py:55-65); Dropout2d is identity in eval."""
    return [E.ConvLayer(ct[0].weight, ct[0].bias, None, pad=1, relu=True, device=device),
            E.ConvLayer(ct[3].weight, ct[3].bias, None, pad=1, relu=True, device=device),
            E.ConvLayer(ct[6].weight, ct[6].bias, None, pad=1, relu=False, device=device)]


def run_cls_tower(layers, feat: E.Act, arena: E.Arena, tag: str = "") -> E.Act:
    """`feat` must carry a fresh lo companion if the first conv runs on the tensor cores."""
    tc = lambda l: l.engine != "simt"
    k1, k2, k3 = layers
    B, h, w, dev = feat.B, feat.H, feat.W, feat.t.device
    a = k1(feat, arena.act(tag + "C1", (B, h, w, k1.Cout), dev, lo=True))
    if tc(k2) and not tc(k1):
        E.split_lo(a)
    a = k2(a, arena.act(tag + "C2", (B, h, w, k2.Cout), dev, lo=True))
    if tc(k3) and not tc(k2):
        E.split_lo(a)
    return k3(a, arena.act(tag + "CLS", (B, h, w, k3.Cout), dev))


def basic_block_runner(blk: M.BasicBlockP, device):
    c1 = E.ConvLayer(blk.conv1.weight, None, E.bn_dict(blk.bn1), stride=blk.stride, pad=1, relu=True, device=device)
    c2 = E.ConvLayer(blk.conv2.weight, None, E.bn_dict(blk.bn2), pad=blk.dilation, dil=blk.dilation, relu=True, device=device)
    return c1, c2


@DETECTOR_DICT.register_module
class Stereo3D(Anchor3DDetector):
    """YOLOStereo3D detector (inference).  `network_cfg` is the reference's `cfg.detector` (R/config/Stereo3D_example:111-167)."""
    N_IMAGES = 2          # images per sample of `launch` (left, right): what pipeline.StreamedInference stages per batch

    def __init__(self, network_cfg):
        super().__init__(network_cfg)
        self.bbox_head = M.StereoHeadP(**self.head_kwargs)
        self.core = M.YoloStereo3DCoreP(dict(network_cfg["backbone"]))

    def build_plan(self, dev) -> dict:
        pl = {}
        pl["backbone"] = ResNetRunner(self.core.backbone, dev)
        neck = self.core.neck
        cv2 = neck.cost_volume_2
        pl["cv2_down"] = E.ConvLayer(cv2.down_sample[0].weight, cv2.down_sample[0].bias, E.bn_dict(cv2.down_sample[1]), relu=True, device=dev)
        w1, b1 = E.fold_bn(cv2.conv3d[0].weight, cv2.conv3d[0].bias, E.bn_dict(cv2.conv3d[1]))     # [F, 2F, 3,3,3]
        w2, b2 = E.fold_bn(cv2.conv3d[3].weight, cv2.conv3d[3].bias, E.bn_dict(cv2.conv3d[4]))
        pl["cv2_w1"] = w1.permute(2, 3, 4, 1, 0).reshape(27, w1.shape[1], w1.shape[0]).contiguous().float().to(dev)
        pl["cv2_b1"] = b1.float().to(dev)
        pl["cv2_w2"] = w2.permute(2, 3, 4, 1, 0).reshape(27, w2.shape[1], w2.shape[0]).contiguous().float().to(dev)
        pl["cv2_b2"] = b2.float().to(dev)
        dr = neck.depth_reasoning
        pl["g4"], pl["bb4"] = GhostRunner(dr.four_to_eight[0], dev), basic_block_runner(dr.four_to_eight[2], dev)
        pl["g8"], pl["bb8"] = GhostRunner(dr.eight_to_sixteen[0], dev), basic_block_runner(dr.eight_to_sixteen[2], dev)
        pl["g16"], pl["bb16"] = GhostRunner(dr.depth_reason[0], dev), basic_block_runner(dr.depth_reason[1], dev)
        ct, rt = self.bbox_head.cls_feature_extraction, self.bbox_head.reg_feature_extraction
        pl["cls"] = cls_tower_runner(ct, dev)
        pl["reg0"] = E.ConvLayer(rt[0].sequence[0].weight, rt[0].sequence[0].bias, E.bn_dict(rt[0].sequence[1]), pad=1, relu=True, device=dev)
        pl["reg_bb"] = basic_block_runner(rt[1], dev)
        pl["reg_out"] = E.ConvLayer(rt[3].weight, rt[3].bias, None, pad=1, relu=False, device=dev)
        return pl

    # ---- forward ------------------------------------------------------------------------------------------
    def core_forward(self, left: torch.Tensor, right: torch.Tensor, reg_out: bool = True, reg_tower: bool = True) -> Tuple[E.Act, E.Act, E.Act]:
        """R/detectors/yolostereo3d_core.py:110-126 + StereoMerging :88-94.  Returns (features, cls_preds, reg_preds) Acts; with
        reg_out=False the last one is the input of the regression output conv (`decode` runs that conv on the rows it reads), with
        reg_tower=False the features again: the regression tower is left to `decode` too (`reg_tower`)."""
        pl = self.prepare()
        ar = self._arena
        dev = left.device
        B, _, H, W = left.shape
        if H % 16 or W % 16:
            raise Vd3dError(f"Stereo3D: image size {H}x{W} must be a multiple of 16")
        if right.shape != left.shape:
            raise Vd3dError(f"Stereo3D: left {tuple(left.shape)} and right {tuple(right.shape)} images differ in shape")
        neck = self.core.neck
        D4, D8, D16 = neck.cost_volume_0.depth_channel, neck.cost_volume_1.depth_channel, neck.cost_volume_2.depth_channel
        h4, w4, h8, w8, h16, w16 = H // 4, W // 4, H // 8, W // 8, H // 16, W // 16
        tc = lambda layer: layer.engine != "simt"
        # scale 4: G4 = cat[vol4 | ghost x1 | ghost x2] (72); scale 8: G8 = cat[bb4(pool G4) | vol8 | ghost x1 | ghost x2]
        G4 = ar.act("G4", (B, h4, w4, 3 * D4), dev, lo=tc(pl["g4"].primary))
        c8 = 3 * D4 + D8
        G8 = ar.act("G8", (B, h8, w8, 3 * c8), dev, lo=tc(pl["g8"].primary))

        def cost_volume_early(f: E.Act, lo_stale: bool) -> bool:
            """PSMCosine of a scale, launched the moment the backbone has produced its features (they are still in L2)."""
            if f.H == h4:
                with self._timed("psm4"):                    # bench.py: CUDA events around the dominant cost-volume kernel, in situ
                    refreshed = E.psm_cosine_stereo(f, B, D4, G4.slice(0, D4), planes_fresh=not lo_stale)
                return lo_stale and not refreshed
            if f.H == h8:
                with self._timed("psm8"):
                    refreshed = E.psm_cosine_stereo(f, B, D8, G8.slice(3 * D4, D8), planes_fresh=not lo_stale)
                return lo_stale and not refreshed
            return lo_stale

        # one [2B] batch: left = [0, B), right = [B, 2B).  The scale-4 / scale-8 features feed only the tensor-core PSMCosine (planes);
        # the scale-16 features are also read as fp32 (left-feature copy, 1x1 down-sample on the SIMT engine)
        bbp = self.core.backbone
        need = [not E.psm_tc_eligible(bbp.out_channels(0), D4), not E.psm_tc_eligible(bbp.out_channels(1), D8), True]
        f4, f8, f16 = pl["backbone"].run([left, right], ar, on_output=cost_volume_early, f32_outputs=need)
        self._hook("feat4", f4), self._hook("feat8", f8), self._hook("feat16", f16)
        self._hook("vol4", G4.slice(0, D4))
        pl["g4"].run(G4)
        c1, c2 = pl["bb4"]
        P8 = E.avgpool2(G4, ar.act("P8", (B, h8, w8, 3 * D4), dev, lo=tc(c1)))
        if tc(c1):
            E.split_lo(P8)
        t = c1(P8, ar.act("T8", (B, h8, w8, 3 * D4), dev, lo=tc(c2)))
        if tc(c2) and not tc(c1):
            E.split_lo(t)
        c2(t, G8.slice(0, 3 * D4), res=P8)
        self._hook("vol8", G8.slice(3 * D4, D8))
        pl["g8"].run(G8)                       # refreshes lo of x = G8[0:96] itself when its primary conv is tensor-core
        c1, c2 = pl["bb8"]
        P16 = E.avgpool2(G8, ar.act("P16", (B, h16, w16, 3 * c8), dev, lo=tc(c1)))
        if tc(c1):
            E.split_lo(P16)
        Fv = neck.cost_volume_2.PSM_features
        c16 = 3 * c8 + Fv * D16
        G16 = ar.act("G16", (B, h16, w16, 3 * c16), dev, lo=True)
        t = c1(P16, ar.act("T16a", (B, h16, w16, 3 * c8), dev, lo=tc(c2)))
        if tc(c2) and not tc(c1):
            E.split_lo(t)
        c2(t, G16.slice(0, 3 * c8), res=P16)
        # scale 16: 1x1 down-sample of left and right in one launch, concat volume fused into the Conv3d pair
        if tc(pl["cv2_down"]) and pl["backbone"].last_lo_stale:
            E.split_lo(f16)
        lr = pl["cv2_down"](f16, ar.act("cv2.lr", (2 * B, h16, w16, Fv), dev))
        mid = ar.get("cv2.mid", (B, D16, h16, w16, Fv), dev)
        vol16 = G16.slice(3 * c8, Fv * D16)
        with self._timed("concat_volume"):
            call("vd3d_concat_volume_conv3d", lr.batch(0, B).ptr, lr.batch(B, 2 * B).ptr, B, h16, w16, Fv, D16,
                 pl["cv2_w1"].data_ptr(), pl["cv2_b1"].data_ptr(), pl["cv2_w2"].data_ptr(), pl["cv2_b2"].data_ptr(),
                 mid.data_ptr(), vol16.ptr, vol16.cs, vol16.co, E._stream())
        self._hook("vol16", vol16)
        pl["g16"].run(G16)                     # x = G16[0:384]: split_lo covers the SIMT-written parts
        cf = f16.C
        FEAT = ar.act("FEAT", (B, h16, w16, cf + 3 * c16), dev, lo=True)
        E.copy_channels(f16.batch(0, B), FEAT.slice(0, cf))
        E.split_lo(FEAT.slice(0, cf))
        c1, c2 = pl["bb16"]
        t = c1(G16, ar.act("T16b", (B, h16, w16, 3 * c16), dev, lo=True))
        if tc(c2) and not tc(c1):
            E.split_lo(t)
        c2(t, FEAT.slice(cf, 3 * c16), res=G16)
        if not tc(c2):
            E.split_lo(FEAT.slice(cf, 3 * c16))
        self._hook("features", FEAT)
        # head towers (R/heads/detection_3d_head.py:509-530); AnchorFlatten == the NHWC layout itself
        cls = run_cls_tower(pl["cls"], FEAT, ar)
        if not reg_tower:
            return FEAT, cls, FEAT
        r0 = pl["reg0"]
        r1 = r0(FEAT, ar.act("R1", (B, h16, w16, r0.Cout), dev, lo=True))
        c1, c2 = pl["reg_bb"]
        if tc(c1) and not tc(r0):
            E.split_lo(r1)
        t = c1(r1, ar.act("R2", (B, h16, w16, c1.Cout), dev, lo=True))
        if tc(c2) and not tc(c1):
            E.split_lo(t)
        r3 = c2(t, ar.act("R3", (B, h16, w16, c2.Cout), dev, lo=True), res=r1)   # block ReLU; the extra nn.ReLU after it is idempotent
        ro = pl["reg_out"]
        if tc(ro) and not tc(c2):
            E.split_lo(r3)
        if not reg_out:
            return FEAT, cls, r3
        reg = self.run_reg_out(ro, r3)
        self._hook("cls_preds", cls), self._hook("reg_preds", reg)
        return FEAT, cls, reg

    def reg_tower(self, pl) -> list:
        """The regression tower in front of reg_out as `decode` takes it: reg0 -> R1, the BasicBlock's c1 -> R2 and c2 (+ R1) -> R3."""
        c1, c2 = pl["reg_bb"]
        return [(pl["reg0"], "R1", None), (c1, "R2", None), (c2, "R3", 0)]

    def launch(self, left, right, P2, P3=None):
        """Enqueue the whole forward (backbone .. NMS) on the current stream; no host synchronisation.
        Returns the DecodeNms object holding the fixed-capacity device outputs."""
        left, right, P2 = self._device_inputs((left, "left"), (right, "right"), (P2, "P2"))
        B, _, H, W = left.shape
        pl = self.prepare()
        ro = pl["reg_out"]
        sparse = self.sparse_reg(ro, B, H // 16, W // 16)
        tower = self.tiled_tower(pl, sparse, H // 16, W // 16)
        _, cls, reg = self.core_forward(left, right, reg_out=not sparse, reg_tower=not tower)
        return self.decode(cls, reg, P2, H, W, reg_out=ro if sparse else None, tower=tower)

    def forward_batch(self, left, right, P2, P3=None):
        """B stereo pairs -> list of B (scores[K], bboxes[K,11], cls_indexes[K]) triples (new API; no reference counterpart).
        One D2H read (the per-image counts) is the only host synchronisation."""
        return self.results(self.launch(left, right, P2, P3))

    def test_forward(self, left_images, right_images, P2, P3=None):
        assert left_images.shape[0] == 1   # reference contract (yolostereo3d_detector.py:78); use forward_batch for B > 1
        return self.forward_batch(left_images, right_images, P2, P3)[0]

    def forward(self, inputs):
        """The reference's stereo list: [left, right, P2, P3] is a test step, five or more elements a training step (raises)."""
        if isinstance(inputs, list) and len(inputs) >= 5:
            return self.train_forward(*inputs)
        return self.test_forward(*inputs)


def build_synthetic_stereo3d(seed: int = 0, depth: int = 34, workdir: Optional[str] = None):
    """Random-init (seeded, de-degenerated) Stereo3D + priors for the bench / smoke / tests: returns
    (detector, state_dict, cfg, (prior_mean, prior_std))."""
    import tempfile
    from .. import synth
    obj_types = ["Car", "Pedestrian"]
    pm, ps = synth.synth_priors(16, 3, obj_types)
    d = workdir or tempfile.mkdtemp(prefix="vd3d_priors_")
    synth.write_priors(d, pm, ps, obj_types)
    cfg = synth.stereo3d_cfg(d, obj_types, depth)
    det = Stereo3D(cfg)
    sd = synth_load(det, seed)
    return det, sd, cfg, (pm, ps)
