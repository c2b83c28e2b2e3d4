"""Host shell shared by the native detectors: the lazily folded / packed weights ("plan"), stage hooks, in-situ kernel timing, decoder
buffers, launch-input checks and the reference's list protocol (`NativeDetector`); and the config parsing, device anchor tables and
batched decode + NMS of the anchor-based 3-D detectors Stereo3D, Yolo3D and GroundAwareYolo3D (`Anchor3DDetector`)."""
from __future__ import annotations

import contextlib
import os

import torch
import torch.nn as nn

from .. import engine as E
from .._lib import Vd3dError
from ..anchors import AnchorTable, load_priors


class NativeDetector(nn.Module):
    """Subclasses hold the parameters, implement `build_plan(dev)` and `launch(images, P2)` -> the decoder holding the fixed-capacity
    device outputs; everything around that lives here."""
    N_IMAGES = 1          # images per sample of `launch` (pipeline.StreamedInference)

    def __init__(self):
        super().__init__()
        self._plan = None
        self._plan_version = None
        self._arena = E.Arena()
        self._decoders = {}
        self._last_decoder = None
        self.stage_hook = None            # tests: callable(name, Act-or-tensor)
        self.profile_events = None        # bench: list collecting (name, start, end) CUDA events of a profiled kernel

    # ---- plan (folded / packed weights) -------------------------------------------------------------------
    def build_plan(self, dev) -> dict:  # pragma: no cover
        raise NotImplementedError

    def prepare(self, force: bool = False):
        """Fold BN into conv weights, pack for the kernels, upload.  Re-run automatically when a parameter or buffer (a BatchNorm running
        statistic) changes; graphs.GraphedStep re-captures on the same version."""
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise Vd3dError(f"{type(self).__name__} has no CPU path: move the module to a CUDA device first")
        ver = (tuple(p._version for p in self.parameters()) + tuple(b._version for b in self.buffers()), str(dev))
        if self._plan is not None and not force and ver == self._plan_version:
            return self._plan
        self._plan, self._plan_version = self.build_plan(dev), ver
        return self._plan

    def _hook(self, name, value):
        if self.stage_hook is not None:
            self.stage_hook(name, value)

    @contextlib.contextmanager
    def _timed(self, name: str):
        """CUDA events around a kernel IN SITU when `profile_events` is a list (bench.py sets it for the timed region; the events are
        recorded on the current stream, nothing synchronises); a no-op otherwise."""
        if self.profile_events is None:
            yield
            return
        e0 = torch.cuda.Event(enable_timing=True)
        e0.record()
        yield
        e1 = torch.cuda.Event(enable_timing=True)
        e1.record()
        self.profile_events.append((name, e0, e1))

    def _decoder(self, key, make):
        """The decoder buffers cached under `key` (built by `make()` on first use); they become `_last_decoder`."""
        if key not in self._decoders:
            self._decoders[key] = make()
        self._last_decoder = self._decoders[key]
        return self._last_decoder

    @staticmethod
    def _device_inputs(*named):
        """(tensor, name) pairs -> the tensors as contiguous float32; a tensor off the GPU is refused by name."""
        for t, name in named:
            E._require_cuda(t, name)
        return [t.float().contiguous() for t, _ in named]

    # ---- detections ---------------------------------------------------------------------------------------
    @staticmethod
    def _result(scores, boxes, cls):
        """One image's triple in the reference's shapes (RetinaNet: 4 box columns; KM3D: cls [K, 1])."""
        return scores, boxes, cls

    def results(self, dec: E.DecodeNms):
        """Per-image (scores, bboxes, cls) triples (one D2H read of the counts)."""
        return [tuple(t.clone() for t in self._result(s, b, c)) for (s, b, c) in dec.results()]

    def forward_batch(self, images, P2=None):
        return self.results(self.launch(images, P2))

    def test_forward(self, img_batch, P2=None):
        assert img_batch.shape[0] == 1   # the reference's test_forward takes one image; use forward_batch for B > 1
        return self.forward_batch(img_batch, P2)[0]

    def train_forward(self, *a, **k):
        raise NotImplementedError("training forward is out of scope of the native inference path (SURVEY.md section 2)")

    def forward(self, inputs):
        """The reference's list protocol: [image, P2] -> one image's triple; a 3-element list is a training step (raises)."""
        if isinstance(inputs, list) and len(inputs) == 3:
            return self.train_forward(*inputs)
        img_batch, P2 = inputs
        return self.test_forward(img_batch, P2)


class Anchor3DDetector(NativeDetector):
    """Subclasses build `self.core` / `self.bbox_head` (parameter holders) and implement `build_plan(dev)` and the forward up to the
    head outputs; the anchors, decode + NMS and post-optimisation live here."""

    def __init__(self, network_cfg):
        super().__init__()
        self.obj_types = network_cfg["obj_types"]
        head = network_cfg["head"]
        acfg = head["anchors_cfg"]
        self.anchors_cfg = {k: acfg[k] for k in ("pyramid_levels", "strides", "sizes", "ratios", "scales")}
        # the remaining arguments of the reference's Anchors (R/heads/anchors.py:11-14) and of the head (detection_3d_head.py:30): honoured
        # or refused, never silently ignored
        y_mm = acfg.get("filter_y_threshold_min_max", (-0.5, 1.8))
        x_thr = acfg.get("filter_x_threshold", 40.0)
        if y_mm is None or x_thr is None:
            raise ValueError("anchors_cfg.filter_y_threshold_min_max / filter_x_threshold must be numbers (set test_cfg.filter_anchor=False to disable the filter)")
        self.anchor_filter = (float(y_mm[0]), float(y_mm[1]), float(x_thr))
        if int(acfg.get("anchor_prior_channel", 6)) != 6:
            raise ValueError("anchors_cfg.anchor_prior_channel must be 6 (z, sin2a, cos2a, w, h, l: the decode layout of detection_3d_head.py:218-263)")
        if not bool(head.get("read_precompute_anchor", True)):
            raise ValueError("head.read_precompute_anchor=False is not supported: the 3-D decode needs the precomputed anchor priors")
        self.num_anchors = len(acfg["pyramid_levels"]) * len(acfg["ratios"]) * len(acfg["scales"])
        self.num_classes = head["num_classes"]
        self.test_cfg = dict(head.get("test_cfg", {}))
        self.filter_anchor = bool(self.test_cfg.get("filter_anchor", head.get("loss_cfg", {}).get("filter_anchor", True)))
        lc = dict(head["layer_cfg"])
        lc.setdefault("num_anchors", self.num_anchors)
        self.layer_cfg = lc
        self.num_cls_output, self.num_reg_output = lc["num_cls_output"], lc["num_reg_output"]
        if self.num_reg_output != 12:
            raise ValueError("num_reg_output must be 12 (decode layout, detection_3d_head.py:218-263)")
        self.head_kwargs = dict(loss_cfg=dict(head.get("loss_cfg", {})),
                                num_regression_loss_terms=head.get("num_regression_loss_terms", 12), **lc)
        self.network_cfg = network_cfg
        n_rows = len(acfg["scales"]) * len(acfg["pyramid_levels"])
        self.prior_mean, self.prior_std = load_priors(head["preprocessed_path"], acfg.get("obj_types", self.obj_types),
                                                      n_rows, len(acfg["ratios"]))
        # R/heads/detection_3d_head.py:294-308 (hill climbing on the yaw, SURVEY.md 8(f).2): device kernel after the NMS (`decode`)
        self.post_optimization = bool(self.test_cfg.get("post_optimization", False))
        self.max_detections = int(self.test_cfg.get("max_candidates", 2048))   # fixed capacity of the decode / NMS stage
        self._anchor_tables = {}

    def _anchor_table(self, H, W, dev) -> AnchorTable:
        key = (H, W, str(dev))
        if key not in self._anchor_tables:
            self._anchor_tables[key] = AnchorTable((H, W), self.anchors_cfg, self.prior_mean, self.prior_std, dev)
        return self._anchor_tables[key]

    # ---- head outputs -> detections -------------------------------------------------------------------------
    def sparse_reg(self, reg_out: E.ConvLayer, B: int, h: int, w: int) -> bool:
        """Run the regression output conv `reg_out` inside `decode`, on the rows the decoder reads only (`ConvLayer.gather`), instead of over
        the whole [B, h, w] map: the inference path, unless a stage hook wants the full `reg_preds` map or VD3D_SPARSE_REG=0.  Only when the
        dense conv takes more than one round of 128-pixel x 128-column tiles on the SMs: a gathered tile walks the whole K loop as a dense one
        does, so a one-round dense conv is as fast (Yolo3D at batch 1, DESIGN §4).  The detections are bit-identical either way."""
        if self.stage_hook is not None or os.environ.get("VD3D_SPARSE_REG", "1") == "0" or not reg_out.gather_ok():
            return False
        dense_tiles = B * -(-h // 8) * -(-w // 16) * -(-reg_out.Cout // 128)
        return dense_tiles > torch.cuda.get_device_properties(reg_out.w_hi.device).multi_processor_count

    def reg_tower(self, pl) -> list:
        """The 3x3 convs at the end of the regression tower that `decode` may run on tile lists (its `tower`); none by default."""
        return []

    @staticmethod
    def tower_tiles_ok(tower, reg_out: E.ConvLayer, h: int, w: int) -> bool:
        """`decode` can run the regression tower `tower` on tile lists over an h x w map: every conv of it and the output conv read their
        input within one pixel (`ConvLayer.tiles_ok`), and the map fits the list builder (`vd3d_reg_tower_tiles`)"""
        return bool(tower) and reg_out.tiles_ok() and all(layer.tiles_ok() for layer, _, _ in tower) and E.tower_tiles_fit(h, w)

    def tiled_tower(self, pl, sparse: bool, h: int, w: int):
        """`decode`'s `tower` for a run with the `sparse_reg` decision `sparse` over an h x w map: `reg_tower(pl)` when it can run on tile
        lists, else () (the caller runs the tower densely)."""
        tower = self.reg_tower(pl) if sparse else []
        return tower if self.tower_tiles_ok(tower, pl["reg_out"], h, w) else ()

    def run_reg_out(self, reg_out: E.ConvLayer, x: E.Act) -> E.Act:
        """The dense regression output conv (R/heads/detection_3d_head.py:509-530): `x` -> reg_preds."""
        return reg_out(x, self._arena.act("REG", (x.B, x.H, x.W, reg_out.Cout), x.t.device))

    def decode(self, cls: E.Act, reg: E.Act, P2: torch.Tensor, H: int, W: int, reg_out: E.ConvLayer = None, tower=()) -> E.DecodeNms:
        """get_anchor + get_bboxes (R/heads/detection_3d_head.py:310-321,341-400), batched, no host sync.  `reg` is the regression map, or
        with `reg_out` (`sparse_reg`) the input of that last conv, which then runs on the (pixel, anchor group) pairs whose anchors pass the
        mask and the score threshold (`vd3d_reg_candidates`, a superset of the rows the decode reads).
        `tower` (with `reg_out`, `tower_tiles_ok`): the convs in front of `reg_out` as (layer, arena name, index of the earlier tower output
        added as residual or None); `reg` is then the tower's input.  Conv j of D runs on the 8 x 16 tiles holding the pixels within D - j
        steps of a candidate pixel (`vd3d_reg_tower_tiles`), which is where `reg_out` reads it through the later convs: bit-identical
        detections, the tower's outputs stale elsewhere."""
        dev = cls.t.device
        B = cls.B
        tab = self._anchor_table(H, W, dev)
        N = tab.N
        mask = self._arena.get("mask", (B, N), dev, dtype=torch.uint8)
        if self.filter_anchor:
            E.anchor_mask(tab.anchors, tab.means_z, P2, mask, *self.anchor_filter)
        else:
            mask.fill_(1)
        self._hook("mask", mask)
        score_thr = self.test_cfg.get("score_thr", 0.5)
        if reg_out is not None:
            A = self.num_anchors
            groups = -(-A // E.REG_GROUP_ANCHORS)
            lst = self._arena.get("reg_list", (groups, B * reg.H * reg.W), dev, dtype=torch.int32)
            counts = self._arena.get("reg_counts", (groups,), dev, dtype=torch.int32)
            pix = self._arena.get("reg_pix", (B, reg.H, reg.W), dev, dtype=torch.uint8) if tower else None
            E.reg_candidates(cls.t, mask, A, self.num_classes, score_thr, lst, counts, pix)
            if tower:
                reg = self._run_tower(tower, reg, pix)
            reg = reg_out.gather(reg, lst, counts, self._arena.act("REG", (B, reg.H, reg.W, reg_out.Cout), dev))
        assert cls.H * cls.W * cls.C == N * self.num_cls_output and reg.C * reg.H * reg.W == N * 12
        assert cls.co == 0 and reg.co == 0 and cls.cs == cls.C and reg.cs == reg.C
        dec = self._decoder((B, str(dev)), lambda: E.DecodeNms(B, self.max_detections, dev))
        dec.run(cls.t.view(B, N, self.num_cls_output), reg.t.view(B, N, 12), tab.anchors, tab.mean_std, mask,
                self.num_classes, score_thr, self.test_cfg.get("nms_iou_thr", 0.5), W, H)
        if self.post_optimization:
            # head.test_cfg.post_optimization (R/heads/detection_3d_head.py:294-308): yaw hill climbing of the kept car boxes deeper than
            # 3 m, in place on the fixed-capacity NMS output, stream-ordered (the reference searches on the CPU with one `.item()` per box)
            dec.post_opt(P2)
        return dec

    def _run_tower(self, tower, x: E.Act, pix: torch.Tensor) -> E.Act:
        """The regression tower (`decode`'s `tower`) on the tile lists built from the candidate pixel map `pix` [B, h, w]."""
        B, h, w, dev = x.B, x.H, x.W, x.t.device
        D = len(tower)
        smaps = self._arena.get("tower_smap", (D, B, h, w), dev, dtype=torch.uint8)
        tiles = self._arena.get("tower_tiles", (D, E.tower_tile_cap(B, h, w), 4), dev, dtype=torch.int32)
        tcount = self._arena.get("tower_count", (D,), dev, dtype=torch.int32)
        E.tower_tiles(pix, smaps, tiles, tcount)
        outs = []
        for j, (layer, name, res) in enumerate(tower):
            d = D - j
            x = layer(x, self._arena.act(name, (B, h, w, layer.Cout), dev, lo=True), res=outs[res] if res is not None else None,
                      tiles=(tiles[d - 1], tcount[d - 1:d], smaps[d - 1]))
            outs.append(x)
        return x


def synth_load(det: nn.Module, seed: int):
    """Fill a detector with the seeded synthetic weights (visualdet3d_b200.synth); returns the state_dict used."""
    from .. import synth
    shapes = {k: tuple(v.shape) for k, v in det.state_dict().items()}
    sd = synth.synth_state_dict(shapes, seed, cls_gain=synth.CLS_GAIN.get(type(det).__name__, 1.6))
    det.load_state_dict(sd, strict=False)
    return sd
