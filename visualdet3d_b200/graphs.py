"""CUDA-graph replay of one detector step.

`GraphedStep` wraps `detector.launch(*images, P2)` [+ `post_forward`] + `pack_records_device` over STATIC device buffers: the first call runs
eagerly (it sizes the arena and builds the anchor tables), the second call captures the same launches into a `torch.cuda.CUDAGraph`, later
calls replay it.  Every launch of the path goes through the C ABI on the current stream and nothing in it synchronises with the host, so
the capture sees exactly the kernels of the eager step and the replay writes the same bits (tests/test_zz_next_rows_gpu.py).
tools/exp_graph.py measures the gain per config (graph replay against eager launches of the same step).
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch

from . import _lib, parallel


class GraphedStep:
    def __init__(self, detector, images: Sequence[torch.Tensor], P2: torch.Tensor, rec_out: torch.Tensor, kmax: int,
                 geometry: bool = False, original_P: Optional[torch.Tensor] = None, pre=None, enabled: bool = True):
        """`images`, `P2`, `original_P`, `rec_out` are the static device buffers the step reads / writes (refill them, then call).
        `pre` = optional callable enqueued in front of the forward inside the same graph (the uint8 input kernel of the pipeline)."""
        for t in list(images) + [P2, rec_out]:
            if not t.is_cuda:
                raise _lib.Vd3dError("GraphedStep: static buffers must live on a CUDA device")
        self.det, self.images, self.P2, self.rec, self.kmax = detector, tuple(images), P2, rec_out, int(kmax)
        self.geometry, self.original_P, self.pre, self.enabled = bool(geometry), original_P, pre, bool(enabled)
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.calls = 0
        self.launches_per_replay = 0
        self.replays = 0
        self._plan_key = None
        self._warm = False
        self.dec = None

    def _eager(self):
        if self.pre is not None:
            self.pre()
        dec = self.det.launch(*self.images, self.P2)
        if self.geometry:
            dec.post_forward(self.P2, self.original_P)
        parallel.pack_records_device(dec, self.kmax, geometry=self.geometry, out=self.rec)
        self.dec = dec
        return dec

    def __call__(self):
        """Enqueue one step on the current stream; returns the DecodeNms object holding the fixed-capacity device outputs."""
        self.calls += 1
        self.det.prepare()                          # re-folds the weights when a parameter changed since the last call (cheap version check otherwise)
        if self._plan_key is not None and getattr(self.det, "_plan_version", None) != self._plan_key:
            self.graph, self._warm = None, False    # parameters changed: the captured pointers / folded weights are stale
        if not self.enabled or getattr(self.det, "stage_hook", None) is not None or getattr(self.det, "profile_events", None) is not None:
            return self._eager()                    # hooks and in-situ event timing need the launches on the stream, not in a graph
        if self.graph is None:
            if not self._warm:
                dec = self._eager()                 # warm-up: sizes the arena, builds anchor tables, sets function attributes
                self._warm, self._plan_key = True, getattr(self.det, "_plan_version", None)
                return dec
            g = torch.cuda.CUDAGraph()
            n0 = _lib.launch_count()
            with torch.cuda.graph(g, capture_error_mode="thread_local"):       # other threads (NCCL watchdog, clock sampler) keep running
                self._eager()
            self.launches_per_replay = _lib.launch_count() - n0
            self.graph = g
        self.graph.replay()
        self.replays += 1
        return self.dec
