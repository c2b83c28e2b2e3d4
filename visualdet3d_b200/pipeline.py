"""Host-fed inference pipeline: pinned host batches -> H2D on a copy stream (double-buffered) -> [uint8 input pipeline] -> forward + NMS
[+ yaw post-optimisation] [+ post-forward geometry] on the compute stream -> ONE all-gather of detection records -> asynchronous D2H into
pinned memory.

The copy of batch i+1 overlaps the forward of batch i, and the host only blocks on the records of batch i-1, so the end-to-end
rate approaches the device-resident rate while every batch still pays its own H2D and D2H inside the timed region.
This is the call a data-loader loop makes (the reference's `scripts/eval.py` loop feeds one frame at a time and synchronises on
every `.cpu()`, R/networks/pipelines/testers.py).

Two input forms:
  * `submit(*images, P2)`          float32 network inputs [B, 3, H, W] (what the reference's dataset + collate_fn produce on the CPU),
  * `submit_frames(*frames, P2)`   uint8 camera frames [B, Hf, Wf, 3]: 4x fewer H2D bytes; ConvertToFloat / CropTop / Resize / Normalize of
                                   the reference's test-time augmentation (R/data/pipeline/stereo_augmentator.py:29-134,213-258) run as one
                                   augmentation kernel launch per camera on the device (csrc/train_augment.cu) right after the copy.
The multi-GPU exchange is off the compute stream: the record block of batch i is gathered on a side stream while batch i+1 computes, so
ranks do not run in lockstep with the slowest GPU (`gather_stream`).
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np
import torch

from . import _lib, parallel
from . import train_augment as ta
from .preprocess import RESIZE_ONLY, RGB_MEAN, RGB_STD


class StreamedInference:
    def __init__(self, detector, batch: int, height: int, width: int, kmax: int = 512, world: int = 1, depth: int = 2,
                 geometry: bool = False, frame_hw: Optional[Sequence[int]] = None, crop_top: int = 0, group=None, graphs: bool = True):
        """`graphs`: replay the forward (.. NMS, post-optimisation, geometry, record block) of every staging slot as ONE CUDA graph from the
        slot's second batch on (`graphs.GraphedStep`; the launches and results are those of the eager step)."""
        n_img = getattr(detector, "N_IMAGES", None)
        if n_img not in (1, 2) or not hasattr(detector, "launch"):
            raise TypeError(f"StreamedInference needs a B200 detector with `launch` and N_IMAGES (got {type(detector).__name__})")
        self.det, self.B, self.kmax, self.world, self.depth, self.n_img = detector, batch, kmax, world, depth, n_img
        self.H, self.W, self.geometry, self.group = height, width, bool(geometry), group
        dev = next(detector.parameters()).device
        self.dev = dev
        self.copy_stream = torch.cuda.Stream(device=dev)
        self.gather_stream = torch.cuda.Stream(device=dev) if world > 1 else None
        mk = lambda *s: torch.empty(*s, device=dev, dtype=torch.float32)
        self.bufs = [tuple(mk(batch, 3, height, width) for _ in range(n_img)) + (mk(batch, 3, 4), mk(batch, 3, 4)) for _ in range(depth)]
        self.rec_width = 1 + kmax * (parallel.REC_GEO if geometry else parallel.REC)
        self.dev_rec = [mk(batch, self.rec_width) for _ in range(depth)]
        self.dev_gathered = [mk(world * batch, self.rec_width) for _ in range(depth)] if world > 1 else None
        self.host_rec = [torch.empty(world * batch, self.rec_width, dtype=torch.float32).pin_memory() for _ in range(depth)]
        self.ev_copied = [torch.cuda.Event() for _ in range(depth)]
        self.ev_free = [torch.cuda.Event() for _ in range(depth)]
        self.ev_packed = [torch.cuda.Event() for _ in range(depth)]
        self.ev_done = [torch.cuda.Event() for _ in range(depth)]
        self.submitted = 0
        self._uncollected = [False] * depth        # slot holds a batch whose records have not been collected yet
        self.h2d_bytes = 4 * (n_img * batch * 3 * height * width + batch * 12)
        self.d2h_bytes = 4 * world * batch * self.rec_width
        self.last_geometry: Optional[list] = None
        self.graphs = bool(graphs)
        self._steps = {}                           # (slot, input form, original_P given) -> graphs.GraphedStep
        # uint8 frame staging (submit_frames)
        self.frame_hw, self.crop_top = (tuple(int(v) for v in frame_hw) if frame_hw is not None else None), int(crop_top)
        if self.frame_hw is not None:
            Hf, Wf = self.frame_hw
            self.frame_bufs = [tuple(torch.empty(batch, Hf, Wf, 3, device=dev, dtype=torch.uint8) for _ in range(n_img)) for _ in range(depth)]
            nb = int(_lib.load().vd3d_train_augment_desc_bytes())
            self._desc_host = [tuple(torch.zeros(batch, nb, dtype=torch.uint8).pin_memory() for _ in range(n_img)) for _ in range(depth)]
            self._desc_dev = [tuple(torch.empty(batch, nb, device=dev, dtype=torch.uint8) for _ in range(n_img)) for _ in range(depth)]
            self._desc_sizes = [None] * depth
            self._mean = np.ascontiguousarray(np.array(RGB_MEAN, dtype=np.float32))
            self._std = np.ascontiguousarray(np.array(RGB_STD, dtype=np.float32))
            self.h2d_bytes_frames = n_img * batch * Hf * Wf * 3 + 4 * batch * 12

    # ---- submission --------------------------------------------------------------------------------------------------------
    def _slot(self):
        i = self.submitted
        k = i % self.depth
        if self._uncollected[k]:
            raise RuntimeError(f"StreamedInference: batch {i - self.depth} has not been collected; at most {self.depth} batches may be in flight")
        return i, k

    def _check_pinned(self, ts):
        for t in ts:
            if t is None:
                continue
            if t.is_cuda or not t.is_pinned():
                raise ValueError("StreamedInference expects pinned host tensors")

    def submit(self, *args, original_P: Optional[torch.Tensor] = None) -> int:
        """Enqueue one batch given as pinned HOST tensors `(*images, P2)` (stereo: left, right, P2; mono: image, P2); returns its ticket.
        Never blocks on the GPU unless `depth` batches are already in flight and uncollected.  The caller's tensors are read by an
        asynchronous DMA: they must stay untouched until `wait_copied(ticket)` returns (a loop that refills the same pinned buffers
        calls it before refilling; P2 / original_P are captured by the same copy, nothing is kept by reference)."""
        if len(args) != self.n_img + 1:
            raise TypeError(f"submit expects {self.n_img} image tensor(s) and P2")
        self._check_pinned(list(args) + [original_P])
        i, k = self._slot()
        cur = torch.cuda.current_stream(self.dev)
        bufs = self.bufs[k]
        with torch.cuda.stream(self.copy_stream):
            if i >= self.depth:
                self.copy_stream.wait_event(self.ev_free[k])       # the forward that last read this staging buffer has consumed it
            for d, h in zip(bufs[:self.n_img + 1], args):
                d.copy_(h, non_blocking=True)
            if original_P is not None:
                bufs[self.n_img + 1].copy_(original_P, non_blocking=True)
            self.ev_copied[k].record(self.copy_stream)
        cur.wait_event(self.ev_copied[k])
        return self._run(i, k, bufs[:self.n_img], bufs[self.n_img], bufs[self.n_img + 1] if original_P is not None else None)

    def submit_frames(self, *args, original_P: Optional[torch.Tensor] = None, sizes: Optional[Sequence[Sequence[int]]] = None) -> int:
        """Enqueue one batch of uint8 camera frames: `(*frames, P2)` with every `frames` a pinned uint8 tensor [B, Hf, Wf, 3] (Hf, Wf =
        `frame_hw` of the constructor; `sizes[b] = (h, w)` marks frames smaller than the staging size, stored top-left) and P2 the
        calibration of the NETWORK input (`preprocess.adjust_calib`).  H2D bytes: 3 per pixel instead of 12."""
        if self.frame_hw is None:
            raise RuntimeError("StreamedInference was built without frame_hw: submit_frames is unavailable")
        if len(args) != self.n_img + 1:
            raise TypeError(f"submit_frames expects {self.n_img} frame tensor(s) and P2")
        self._check_pinned(list(args) + [original_P])
        Hf, Wf = self.frame_hw
        for f in args[:self.n_img]:
            if f.dtype != torch.uint8 or tuple(f.shape) != (self.B, Hf, Wf, 3):
                raise ValueError(f"frames must be uint8 [{self.B}, {Hf}, {Wf}, 3]")
        i, k = self._slot()
        cur = torch.cuda.current_stream(self.dev)
        bufs, fb = self.bufs[k], self.frame_bufs[k]
        key = tuple(tuple(int(v) for v in s) for s in sizes) if sizes is not None else None
        new_desc = self._desc_sizes[k] is None or self._desc_sizes[k] != ("u", key)
        if new_desc:
            for c in range(self.n_img):
                dh = self._desc_host[k][c].numpy()
                for b in range(self.B):
                    h, w = (key[b] if key is not None else (Hf, Wf))          # stored top-left in the Wf-wide staging frame
                    dh[b] = ta._describe(fb[c][b].data_ptr(), (h, w, 3), crop_top=self.crop_top, out_hw=(self.H, self.W), pitch=Wf * 3,
                                         **RESIZE_ONLY)
        with torch.cuda.stream(self.copy_stream):
            if i >= self.depth:
                self.copy_stream.wait_event(self.ev_free[k])
            for d, h in zip(fb, args[:self.n_img]):
                d.copy_(h, non_blocking=True)
            bufs[self.n_img].copy_(args[self.n_img], non_blocking=True)
            if original_P is not None:
                bufs[self.n_img + 1].copy_(original_P, non_blocking=True)
            if new_desc:
                for c in range(self.n_img):
                    self._desc_dev[k][c].copy_(self._desc_host[k][c], non_blocking=True)
                self._desc_sizes[k] = ("u", key)
            self.ev_copied[k].record(self.copy_stream)
        cur.wait_event(self.ev_copied[k])
        for c in range(self.n_img):          # test-time augmentation on the device: uint8 HWC -> cropped, resized, normalised float32 CHW
            _lib.call("vd3d_train_augment", self._desc_dev[k][c].data_ptr(), self.B, 3, self.H, self.W, ta._vp(self._mean), ta._vp(self._std),
                      bufs[c].data_ptr(), cur.cuda_stream)
        return self._run(i, k, bufs[:self.n_img], bufs[self.n_img], bufs[self.n_img + 1] if original_P is not None else None)

    def _run(self, i: int, k: int, images, P2, original_P) -> int:
        cur = torch.cuda.current_stream(self.dev)
        from .graphs import GraphedStep
        key = (k, original_P is not None)
        if key not in self._steps:
            self._steps[key] = GraphedStep(self.det, images, P2, self.dev_rec[k], self.kmax, geometry=self.geometry, original_P=original_P,
                                           enabled=self.graphs)
        with torch.no_grad():
            # backbone .. NMS (+ the yaw post-optimisation when the detector's test_cfg asks for it) [+ geometry] + the record block
            self._steps[key]()
        rec = self.dev_rec[k]
        self.ev_free[k].record(cur)
        if self.world > 1:
            # the single collective of the path, on a side stream: the next forward does not wait for the slowest rank's records
            self.ev_packed[k].record(cur)
            with torch.cuda.stream(self.gather_stream):
                self.gather_stream.wait_event(self.ev_packed[k])
                g = parallel.all_gather_records(rec, group=self.group, out=self.dev_gathered[k])
                self.host_rec[k].copy_(g, non_blocking=True)
                self.ev_done[k].record(self.gather_stream)
        else:
            self.host_rec[k].copy_(rec, non_blocking=True)
            self.ev_done[k].record(cur)
        self._uncollected[k] = True
        self.submitted += 1
        return i

    def wait_copied(self, ticket: int) -> None:
        """Block until the H2D copies of batch `ticket` have completed: the caller's pinned buffers may then be refilled."""
        if not (self.submitted - self.depth <= ticket < self.submitted):
            raise RuntimeError(f"StreamedInference: ticket {ticket} is not in flight")
        self.ev_copied[ticket % self.depth].synchronize()

    # ---- collection --------------------------------------------------------------------------------------------------------
    def collect(self, ticket: int) -> List:
        """Block until batch `ticket` is on the host; returns the per-image (scores, boxes, classes) of the GLOBAL batch.  With
        `geometry=True` the post-forward columns of the same batch are left in `self.last_geometry` (per image: box3d [K, 7] in the
        camera frame, theta [K], box2d [K, 4] in original-frame pixels) and `kitti_text` formats them."""
        k = ticket % self.depth
        if not (self.submitted - self.depth <= ticket < self.submitted) or not self._uncollected[k]:
            raise RuntimeError(f"StreamedInference: ticket {ticket} is not in flight")
        self.ev_done[k].synchronize()
        self._uncollected[k] = False
        geo = [] if self.geometry else None
        try:
            res = parallel.unpack_records(self.host_rec[k], parallel.REC_GEO if self.geometry else parallel.REC, geo)
        except _lib.Vd3dError:
            from .engine import fp16_range_overflowed
            fp16_range_overflowed(reset=True)          # fp16-range guard tripped: clear the sticky device flag, then report
            raise
        self.last_geometry = geo
        return res

    def kitti_text(self, results, class_names: Sequence[str], threshold: float = 0.4) -> List[str]:
        """KITTI result text of every image of the batch just collected (write_result_to_file, R/data/kitti/utils.py:162-201), from
        the device-computed geometry: the host only formats."""
        if not self.geometry or self.last_geometry is None:
            raise RuntimeError("kitti_text needs geometry=True and a collected batch")
        from . import postforward as pf
        out = []
        for (s, b, c), (box3d, theta, box2d) in zip(results, self.last_geometry):
            out.append(pf.kitti_lines(s, box2d, box3d, theta, [class_names[int(i)] for i in c], threshold))
        return out
