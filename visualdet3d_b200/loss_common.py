"""Host-side helpers shared by the GPU training losses (anchor_loss, retina_loss, monoflex_loss, km3d_loss, disparity_loss): the host
counterpart of csrc/loss_common.cuh.  Input checks raise before any launch; nothing here synchronises the host."""
from __future__ import annotations

import ctypes
from typing import Mapping

import torch

from . import _lib


def check(t, who: str, name: str, dtypes) -> None:
    """Refuse anything but a CUDA tensor of one of `dtypes` (a dtype or a tuple of them), naming the loss `who` and the input `name`.
    A tensor of the wrong dtype is refused for its dtype before its device is looked at."""
    dtypes = dtypes if isinstance(dtypes, tuple) else (dtypes,)
    if isinstance(t, torch.Tensor) and t.dtype not in dtypes:
        raise RuntimeError(f"{who}: {name} must be {' or '.join(str(d) for d in dtypes)}, got {t.dtype}")
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError(f"{who}: {name} must be a CUDA tensor (there is no CPU path)")


def stream(t: torch.Tensor) -> int:
    """The handle of the current CUDA stream of t's device, for the library's `stream` argument."""
    return torch.cuda.current_stream(t.device).cuda_stream


def ptr_array(ts):
    """Host array of device pointers (the C ABI's maps / targets / grads)."""
    return (ctypes.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


def workspace(entry: str, *sizes, device):
    """(uint8 device buffer, its size in bytes) for the library's workspace query `entry` at `sizes`; raises Vd3dError with the library's
    message when the query refuses the sizes.  The buffer holds at least one byte: the library refuses a null workspace."""
    lib = _lib.load()
    n = int(getattr(lib, entry)(*sizes))
    if n < 0:
        raise _lib.Vd3dError(f"{entry} failed ({n}): {lib.vd3d_last_error().decode()}")
    return torch.empty(max(n, 1), dtype=torch.uint8, device=device), n


def as_config(config_cls, cfg, *args):
    """cfg itself when it is a `config_cls`, else config_cls.from_loss_cfg(cfg, *args) (cfg: a head's loss_cfg mapping)."""
    return cfg if isinstance(cfg, config_cls) else config_cls.from_loss_cfg(cfg, *args)


def cached_on(obj, attr: str, key, build):
    """build(), cached in obj.__dict__[attr] until `key` changes."""
    cached = obj.__dict__.get(attr)
    if cached is None or cached[0] != key:
        cached = (key, build())
        obj.__dict__[attr] = cached
    return cached[1]


def grad_out_pair(g_a, g_b, device) -> torch.Tensor:
    """The [2] float32 grad_output of a loss pair's backward: autograd passes None for an output that no gradient reached (zero)."""
    zero = torch.zeros(1, dtype=torch.float32, device=device)
    return torch.cat([(zero if g_a is None else g_a.reshape(1)), (zero if g_b is None else g_b.reshape(1))]).float()


def map_inputs(who: str, head: str, maps, hm_targets, row_targets, max_rows: int, output: Mapping, annotations: Mapping, P2: torch.Tensor):
    """Validated, contiguous (maps, targets, sizes (B, C, H, W, K)) of a CenterNet-style head loss; raises before any launch.

    maps: (name, channels or None) of output's [B, C, H, W] float32 maps, the first (hm) setting B, C, H, W.  hm_targets: (name, channels
    or None for C) of the float32 [B, ch, H, W] heatmap targets.  row_targets: (name, dtypes, trailing shape, rows per object) of the
    per-object targets, [B, K * rows per object, *trailing shape] with K = annotations['ind'].shape[1] <= max_rows.  The targets come
    back in that order, heatmaps first and P2 [B, 3, 4] last."""
    out = []
    for name, ch in maps:
        t = output[name]
        check(t, who, f"output['{name}']", torch.float32)
        if t.dim() != 4:
            raise ValueError(f"{who}: output['{name}'] must be [B, C, H, W], got {tuple(t.shape)}")
        if ch is not None and t.shape[1] != ch:
            raise ValueError(f"{who}: output['{name}'] has {t.shape[1]} channels, the {head} head has {ch}")
        out.append(t.contiguous())
    B, C, H, W = out[0].shape
    for (name, _), t in zip(maps, out):
        if (t.shape[0], t.shape[2], t.shape[3]) != (B, H, W):
            raise ValueError(f"{who}: output['{name}'] {tuple(t.shape)} does not match hm's B, H, W = {(B, H, W)}")
    targets = []
    for name, ch in hm_targets:
        t = annotations[name]
        check(t, who, f"annotations['{name}']", torch.float32)
        expected = (B, C if ch is None else ch, H, W)
        if tuple(t.shape) != expected:
            raise ValueError(f"{who}: annotations['{name}'] {tuple(t.shape)}, expected {expected}")
        targets.append(t.contiguous())
    ind = annotations["ind"]
    if ind.dim() != 2 or ind.shape[0] != B:
        raise ValueError(f"{who}: annotations['ind'] {tuple(ind.shape)}, expected [{B}, K]")
    K = ind.shape[1]
    if not 1 <= K <= max_rows:
        raise ValueError(f"{who}: {K} object rows per image, 1..{max_rows} supported")
    for name, dtypes, trail, per in row_targets:
        t = annotations[name]
        check(t, who, f"annotations['{name}']", dtypes)
        if tuple(t.shape) != (B, K * per) + trail:
            raise ValueError(f"{who}: annotations['{name}'] {tuple(t.shape)}, expected {(B, K * per) + trail}")
        targets.append(t.contiguous())
    check(P2, who, "P2", torch.float32)
    if tuple(P2.shape) != (B, 3, 4):
        raise ValueError(f"{who}: P2 {tuple(P2.shape)}, expected {(B, 3, 4)}")
    targets.append(P2.contiguous())
    return out, targets, (B, C, H, W, K)
