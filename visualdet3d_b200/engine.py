"""Host-side execution engine: activation views, weight folding / packing and thin launchers over the C ABI.

PyTorch is used for device memory and streams only; every arithmetic op on the path is a kernel of
libvd3d_b200.so.  Activations are fp32 NHWC; an `Act` is a channel slice [co, co+C) of a [B,H,W,cs] tensor, which
is how every torch.cat of the reference is fused away (producers write straight into their slice).
"""
from __future__ import annotations

import ctypes
from typing import Dict, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from ._lib import call


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _require_cuda(t: torch.Tensor, what: str):
    if not t.is_cuda:
        raise _lib.Vd3dError(f"{what}: tensor is on {t.device}; the B200 path has no CPU fallback")


class Act:
    """Channel slice [co, co+C) of an NHWC fp32 tensor `t` of shape [B, H, W, cs].

    `lo` (optional) is the tensor-core companion of `t`, in one of two forms:
      * float32, same shape as `t`:  t - (t & 0xFFFFE000), the part of every value the tf32 MMA does not see ("tc" engine);
      * float16, shape [2, B, H, W, cs]: planes hi = rn16(t) and lo = rn16(t - hi) ("tc16" engine, the default).
    The wgmma conv engine consumes and produces these; other producers leave them stale and the plan calls `split_lo`
    before a tensor-core consumer."""
    __slots__ = ("t", "co", "C", "lo", "f32", "lo_fresh", "valid")

    def __init__(self, t: torch.Tensor, co: int = 0, C: Optional[int] = None, lo: Optional[torch.Tensor] = None, f32: bool = True):
        assert t.dim() == 4 and t.dtype == torch.float32 and t.is_contiguous()
        self.t, self.co, self.lo = t, co, lo
        # False: the fp32 tensor was NOT written by the producer (planes-only output of a tensor-core conv whose consumers are all
        # tensor-core convs / plane residuals): the fp16 (hi, lo) planes are the tensor, `t` only carries the shape
        self.f32 = f32
        self.lo_fresh = False      # True once a kernel that writes the companion together with the tensor (tensor-core conv, fused DCN, row conv) produced THIS view
        self.valid = None          # [B, H, W] uint8 map of the pixels the producer wrote (a tile-listed conv); None: every pixel
        self.C = (t.shape[3] - co) if C is None else C
        assert 0 <= co and co + self.C <= t.shape[3]
        assert lo is None or (lo.dtype == torch.float32 and lo.shape == t.shape) or \
            (lo.dtype == torch.float16 and tuple(lo.shape) == (2,) + tuple(t.shape))

    B = property(lambda s: s.t.shape[0])
    H = property(lambda s: s.t.shape[1])
    W = property(lambda s: s.t.shape[2])
    cs = property(lambda s: s.t.shape[3])

    def slice(self, co: int, C: int) -> "Act":
        return Act(self.t, self.co + co, C, self.lo, self.f32)

    def batch(self, b0: int, b1: int) -> "Act":
        # (a batch sub-range of the fp16 planes is not contiguous: such views drop the companion; they only feed non-TC kernels)
        lo = self.lo[b0:b1] if (self.lo is not None and self.lo.dtype == torch.float32) else None
        need_f32(self, "Act.batch")
        return Act(self.t[b0:b1], self.co, self.C, lo)

    @property
    def lo_ptr(self):
        """fp32 lo companion pointer (None when absent or in fp16-plane form)."""
        return self.lo.data_ptr() if (self.lo is not None and self.lo.dtype == torch.float32) else None

    @property
    def h16(self) -> bool:
        return self.lo is not None and self.lo.dtype == torch.float16

    @property
    def h16_ptrs(self):
        return (self.lo[0].data_ptr(), self.lo[1].data_ptr()) if self.h16 else (None, None)

    @property
    def ptr(self) -> int:
        return self.t.data_ptr()

    def to_nchw(self) -> torch.Tensor:
        """Dense [B, C, H, W] copy (tests / NCHW-facing op mirrors)."""
        if not self.f32:        # planes-only tensor: value = hi + lo (test / hook path: plain torch ops)
            v = self.lo[0][..., self.co:self.co + self.C].float() + self.lo[1][..., self.co:self.co + self.C].float()
            return v.permute(0, 3, 1, 2).contiguous()
        out = torch.empty(self.B, self.C, self.H, self.W, device=self.t.device, dtype=torch.float32)
        call("vd3d_nhwc_to_nchw", self.ptr, out.data_ptr(), self.B, self.C, self.H, self.W, self.cs, self.co, _stream())
        return out


def need_f32(x: "Act", what: str):
    """Plan check: `what` reads the fp32 tensor of `x`, which a planes-only producer did not write."""
    if not x.f32:
        raise _lib.Vd3dError(f"{what}: the activation exists only as fp16 (hi, lo) planes (plan bug: its producer was told no fp32 consumer follows)")


def planes_mode_ok() -> bool:
    """Planes-only activations between tensor-core convs (`vd3d_conv2d_tc16` with no fp32 output): default on with the fp16-split engine;
    VD3D_PLANES=0 restores the round-1 behaviour (every conv also writes the fp32 tensor)."""
    import os
    return conv_engine_default() == "tc16" and os.environ.get("VD3D_PLANES", "1") != "0"


def planes_only_ok(layer) -> bool:
    """this tensor-core layer may write its output as planes only (no fp32 copy): planes mode on and the tile not wider than
    VD3D_PLANES_MAXC columns (default 160: the widest epilogue variant, 16 x 8 accumulator groups per thread, has no registers to spare
    for the planes form and runs slower with it)"""
    import os
    return planes_mode_ok() and layer.engine == "tc16" and layer.Cout <= int(os.environ.get("VD3D_PLANES_MAXC", "160"))


class Arena:
    """Named, shape-keyed device buffers: allocated once, pointer-stable across forwards (CUDA-graph friendly)."""

    def __init__(self, lo_form: Optional[str] = None):
        self._bufs: Dict[Tuple, torch.Tensor] = {}
        self.lo_form = lo_form or lo_mode()      # companion form is fixed when the owning detector is built

    def get(self, name: str, shape: Sequence[int], device, dtype=torch.float32, zero: bool = False) -> torch.Tensor:
        key = (name, tuple(int(s) for s in shape), str(device), dtype)
        t = self._bufs.get(key)
        if t is None:
            t = (torch.zeros if zero else torch.empty)(key[1], device=device, dtype=dtype)
            self._bufs[key] = t
        return t

    def act(self, name: str, shape: Sequence[int], device, lo: bool = False, zero: bool = False) -> Act:
        """NHWC activation buffer (optionally with its `lo` companion for the tensor-core engine)."""
        t = self.get(name, shape, device, zero=zero)
        if not lo:
            return Act(t)
        if self.lo_form == "h16":
            return Act(t, 0, None, self.get(name + "#h16", (2,) + tuple(shape), device, dtype=torch.float16, zero=True))
        return Act(t, 0, None, self.get(name + "#lo", shape, device, zero=True))

    def level_acts(self, name: str, B: int, hws: Sequence[Tuple[int, int]], C: int, device, lo: bool = False) -> list:
        """One NHWC activation per (H, W) in `hws`, as views of ONE allocation per form with the levels concatenated ([B, H, W, C] blocks in
        order; the fp16 planes likewise): the layout `ConvLayer.run_levels` writes and reads."""
        sizes = [B * h * w * C for h, w in hws]
        t = self.get(name, (sum(sizes),), device)
        p = self.get(name + "#h16", (2, sum(sizes)), device, dtype=torch.float16, zero=True) if lo and self.lo_form == "h16" else None
        if lo and p is None:
            raise _lib.Vd3dError("Arena.level_acts: the concatenated form needs the fp16 (hi, lo) planes (engine tc16)")
        out, o = [], 0
        for (h, w), n in zip(hws, sizes):
            out.append(Act(t[o:o + n].view(B, h, w, C), 0, None, p[:, o:o + n].view(2, B, h, w, C) if p is not None else None))
            o += n
        return out

    def nbytes(self) -> int:
        return sum(t.numel() * t.element_size() for t in self._bufs.values())


# -------------------------------------------------------------------------------------------------------------
# weight folding / packing (host, float64 -> float32)
# -------------------------------------------------------------------------------------------------------------
def fold_bn(weight: torch.Tensor, bias: Optional[torch.Tensor], bn: Optional[Dict[str, torch.Tensor]], eps: float = 1e-5):
    """conv (+bias) followed by eval-mode BatchNorm -> (weight', bias') in float64.
    y = (conv(x) + b - mean) * gamma / sqrt(var + eps) + beta."""
    w = weight.detach().double().cpu()
    b = bias.detach().double().cpu() if bias is not None else torch.zeros(w.shape[0], dtype=torch.float64)
    if bn is not None:
        scale = bn["weight"].detach().double().cpu() / torch.sqrt(bn["running_var"].detach().double().cpu() + eps)
        w = w * scale.view(-1, *([1] * (w.dim() - 1)))
        b = (b - bn["running_mean"].detach().double().cpu()) * scale + bn["bias"].detach().double().cpu()
    return w, b


def bn_dict(mod) -> Dict[str, torch.Tensor]:
    return dict(weight=mod.weight, bias=mod.bias, running_mean=mod.running_mean, running_var=mod.running_var)


def conv_engine_default() -> str:
    """'tc16' = wgmma fp16-split engine (3 kind::f16 MMAs, default), 'tc' = wgmma 3xTF32 engine, 'simt' = exact-fp32 SIMT
    engine everywhere, 'tc1' = single-pass TF32 (NOT parity-grade; diagnostics only)."""
    import os
    return os.environ.get("VD3D_CONV_ENGINE", "tc16")


def lo_mode() -> str:
    """form of the tensor-core companions allocated by Arena.act: 'h16' (fp16 hi/lo planes) or 'f32' (tf32 lo tensor)"""
    return "h16" if conv_engine_default() == "tc16" else "f32"


def fp16_split(w: torch.Tensor):
    """w (float32/64, already scaled into fp16 range) -> (hi, lo) fp16 with hi = rn16(w), lo = rn16(w - hi)."""
    w = w.float()
    hi = w.half()
    lo = (w - hi.float()).half()
    return hi.contiguous(), lo.contiguous()


def fp16_split_scaled(w: torch.Tensor):
    """Packed float64 weight matrix -> (w_hi, w_lo, out_scale): w * S split by `fp16_split`, S = 2^k the power of two that puts max |w| * S in
    [8192, 16384) (k clamped to [-24, 24]; 0 for an all-zero matrix) so that the lo parts stay normal fp16 numbers; out_scale = 1 / S (exact)."""
    wmax = float(w.abs().max())
    k = int(np.floor(np.log2(16384.0 / wmax))) if wmax > 0 else 0
    k = max(-24, min(24, k))
    hi, lo = fp16_split(w * (2.0 ** k))
    return hi, lo, float(2.0 ** (-k))


def tf32_split(w: torch.Tensor):
    """w (float32) -> (hi, lo) with hi = w & 0xFFFFE000 (the bits the tf32 MMA reads) and lo = tf32-truncated (w - hi)."""
    wi = w.contiguous().view(torch.int32)
    hi = (wi & -8192).view(torch.float32)
    lo = ((w - hi).contiguous().view(torch.int32) & -8192).view(torch.float32)
    return hi.contiguous(), lo.contiguous()


class ConvLayer:
    """A dense conv with everything after it fused: folded BN, bias, optional residual, optional ReLU.
    SIMT engine weights are packed [KH*KW*Cin_pad][Cout] (k = (kh*KW + kw)*Cin_pad + ci); tensor-core engine weights
    [Cout][KH*KW*Cin] (K contiguous) as a (hi, lo) pair."""

    def __init__(self, weight, bias=None, bn=None, stride=1, pad=0, dil=1, relu=False, device="cuda", cin_pad: Optional[int] = None,
                 engine: Optional[str] = None):
        w, b = fold_bn(weight, bias, bn)
        Cout, Cin, KH, KW = w.shape
        cin_p = cin_pad or Cin
        if cin_p != Cin:
            wp = torch.zeros(Cout, cin_p, KH, KW, dtype=torch.float64)
            wp[:, :Cin] = w
            w = wp
        self.Cin, self.Cout, self.KH, self.KW = cin_p, Cout, KH, KW
        self.stride, self.pad, self.dil, self.relu = stride, pad, dil, relu
        eng = engine or conv_engine_default()
        on_gpu = str(device).startswith("cuda")
        if eng == "tc16":      # fp16-split engine: any stride <= 4, Cin % 8 (zero-filled up to the 64-channel k-block), Cout % 4;
            # below 32 input channels the 64-channel k-block is mostly padding and the SIMT engine is faster
            import os
            eligible = on_gpu and stride <= 4 and cin_p % 8 == 0 and cin_p >= int(os.environ.get("VD3D_TC_MINC", "32")) and Cout % 4 == 0 and Cout >= 16
        else:
            eligible = on_gpu and stride == 1 and cin_p % 32 == 0 and Cout % 16 == 0
        self.engine = eng if (eng in ("tc", "tc1", "tc16") and eligible) else "simt"
        self.b = b.float().to(device)
        self.w = self.w_hi = self.w_lo = None
        self.out_scale = 1.0
        if self.engine == "simt":
            self.w = w.permute(2, 3, 1, 0).reshape(KH * KW * cin_p, Cout).contiguous().float().to(device)
        elif self.engine == "tc16":
            cin64 = (cin_p + 63) // 64 * 64
            wk = torch.zeros(Cout, KH * KW, cin64, dtype=torch.float64)
            wk[:, :, :cin_p] = w.permute(0, 2, 3, 1).reshape(Cout, KH * KW, cin_p)
            hi, lo, self.out_scale = fp16_split_scaled(wk.reshape(Cout, KH * KW * cin64))
            self.w_hi, self.w_lo = hi.to(device), lo.to(device)
            self.bn_tile = 0          # 0 = the library's policy for the engine in use (vd3d_tc_pick_bn_persistent / vd3d_tc_pick_bn)
            self.passes = 3           # 2 = error-budget experiments (tools/error_budget.py): drop the A_lo * W_hi product
        else:
            wk = w.permute(0, 2, 3, 1).reshape(Cout, KH * KW * cin_p).contiguous().float()
            hi, lo = tf32_split(wk)
            self.w_hi, self.w_lo = hi.to(device), lo.to(device)
            self.bn_tile = int(_lib.load().vd3d_tc_pick_bn(Cout))

    def out_hw(self, H, W):
        Ho = (H + 2 * self.pad - self.dil * (self.KH - 1) - 1) // self.stride + 1
        Wo = (W + 2 * self.pad - self.dil * (self.KW - 1) - 1) // self.stride + 1
        return Ho, Wo

    def _check_tc16_input(self, x: Act, what: str):
        if self.engine != "tc16" or getattr(self, "passes", 3) != 3:
            raise _lib.Vd3dError(f"{what}: only the fp16-split tensor-core engine (VD3D_CONV_ENGINE=tc16) runs it")
        if not x.h16:
            raise _lib.Vd3dError(f"{what}: input activation has no fp16 (hi, lo) planes (plan bug: missing split_lo)")
        if CHECK_LO:
            check_lo(x)

    def _tc16(self, xs: Sequence[Act], outs: Sequence[Act], res: Optional[Sequence[Act]], res_up: bool, relu: bool, f32_out: bool):
        """One vd3d_conv2d_tc16 launch: outs[l] = conv(xs[l]) [+ res[l]] for every level l.  The residual is read from its fp32 tensor when that
        is valid, else from its fp16 planes; res_up: it has half the output size and is added nearest-upsampled.  f32_out=False writes the
        output planes only."""
        L = len(xs)
        P, I = ctypes.c_void_p * L, ctypes.c_int * L        # per-level arrays

        def planes(acts):
            ps = [a.h16_ptrs for a in acts]
            return P(*[h for h, _ in ps]), P(*[lo for _, lo in ps])
        o, r0 = outs[0], res[0] if res is not None else None
        xh, xl = planes(xs)
        oh, ol = planes(outs) if o.h16 else (None, None)
        rh, rl = planes(res) if r0 is not None and not r0.f32 else (None, None)
        call("vd3d_conv2d_tc16", L, xh, xl, I(*[x.H for x in xs]), I(*[x.W for x in xs]), xs[0].B, self.Cin, xs[0].cs, xs[0].co,
             self.w_hi.data_ptr(), self.w_lo.data_ptr(), self.out_scale, self.b.data_ptr(), self.KH, self.KW, self.pad, self.dil, self.stride,
             P(*[r.ptr for r in res]) if r0 is not None and r0.f32 else None, rh, rl,
             I(*[r.H for r in res]) if res_up else None, I(*[r.W for r in res]) if res_up else None,
             r0.cs if r0 is not None else 0, r0.co if r0 is not None else 0,
             P(*[t.ptr for t in outs]) if f32_out else None, oh, ol, self.Cout, o.cs, o.co, 1 if relu else 0, self.passes, self.bn_tile, _stream())

    def _tc16_tiles(self, x: Act, out: Act, res: Optional[Act], relu: bool, f32_out: bool, tiles):
        """One vd3d_conv2d_tc16_tiles launch (the `tiles` form of `__call__`)."""
        lst, cnt, smap = tiles
        assert self.tiles_ok() and lst.dtype == cnt.dtype == torch.int32 and smap.dtype == torch.uint8 and lst.shape[-1] == 4
        assert lst.is_contiguous() and smap.is_contiguous() and tuple(smap.shape) == (x.B, x.H, x.W)
        oh, ol = out.h16_ptrs if out.h16 else (None, None)
        rf = res is not None and res.f32
        rh, rl = res.h16_ptrs if res is not None and not rf else (None, None)
        xh, xl = x.h16_ptrs
        call("vd3d_conv2d_tc16_tiles", xh, xl, x.B, x.H, x.W, self.Cin, x.cs, x.co, self.w_hi.data_ptr(), self.w_lo.data_ptr(), self.out_scale,
             self.b.data_ptr(), self.KH, self.KW, self.pad, self.dil, res.ptr if rf else None, rh, rl,
             res.cs if res is not None else 0, res.co if res is not None else 0,
             out.ptr if f32_out else None, oh, ol, self.Cout, out.cs, out.co, 1 if relu else 0, self.bn_tile,
             lst.data_ptr(), cnt.data_ptr(), smap.data_ptr(), _stream())

    def gather_ok(self) -> bool:
        """`gather` runs this layer: fp16-split engine, stride 1, an output of the input's size"""
        return self.engine == "tc16" and self.passes == 3 and self.stride == 1 and 2 * self.pad == self.dil * (self.KH - 1) == self.dil * (self.KW - 1)

    def tiles_ok(self) -> bool:
        """`__call__` with `tiles` runs this layer: a 3x3 / pad 1 / stride 1 conv of the fp16-split engine (each output pixel reads its input
        within one pixel)"""
        return self.gather_ok() and self.KH == self.KW == 3 and self.pad == self.dil == 1

    def gather(self, x: Act, lst: torch.Tensor, counts: torch.Tensor, out: Act) -> Act:
        """The conv (with its bias, no ReLU) at the listed output pixels only, one 96-column group of `out` at a time
        (`vd3d_conv2d_tc16_gather`): `lst` [groups, B * H * W] int32 holds counts[g] pixels b * H * W + h * W + w for group g.  Bit-identical
        to the dense conv there; every other element of `out` is left as it was."""
        assert self.gather_ok() and not self.relu and x.C == self.Cin and out.C == self.Cout and (out.B, out.H, out.W) == (x.B, x.H, x.W)
        self._check_tc16_input(x, "gathered conv")
        xh, xl = x.h16_ptrs
        call("vd3d_conv2d_tc16_gather", xh, xl, x.B, x.H, x.W, self.Cin, x.cs, x.co, self.w_hi.data_ptr(), self.w_lo.data_ptr(), self.out_scale,
             self.b.data_ptr(), self.KH, self.KW, self.pad, self.dil, lst.data_ptr(), counts.data_ptr(), counts.shape[0],
             out.ptr, self.Cout, out.cs, out.co, _stream())
        out.f32 = True
        return out

    def run_levels(self, xs: Sequence[Act], outs: Sequence[Act], res: Optional[Sequence[Act]] = None, res_up: bool = False):
        """The conv on several tensors of different sizes in ONE persistent launch (vd3d_conv2d_tc16 over L levels): outs[l] = conv(xs[l])
        [+ res[l], nearest-upsampled when res_up].  Each form of `outs` (fp32, fp16 planes) and `res` must be views of one allocation with the
        levels concatenated (`Arena.level_acts`).  Bit-identical to calling the layer on every level."""
        L = len(xs)
        assert 1 <= L == len(outs) and (res is None or len(res) == L)
        for x, o in zip(xs, outs):
            self._check_tc16_input(x, "multi-level conv")
            assert x.C == self.Cin and o.C == self.Cout and o.B == x.B and (o.H, o.W) == self.out_hw(x.H, x.W) and o.h16 == outs[0].h16
            assert (x.cs, x.co, o.cs, o.co) == (xs[0].cs, xs[0].co, outs[0].cs, outs[0].co)
        if res is not None:
            for r in res:
                need_f32(r, "multi-level conv residual")
        self._tc16(xs, outs, res, res_up and res is not None, self.relu, True)
        for o in outs:
            o.f32, o.lo_fresh = True, o.h16
        return outs

    def __call__(self, x: Act, out: Act, res: Optional[Act] = None, relu: Optional[bool] = None, f32_out: bool = True, res_up: bool = False,
                 tiles: Optional[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]] = None):
        """f32_out=False (fp16-split engine only): write ONLY the fp16 (hi, lo) planes of the output; legal when every consumer is a
        tensor-core conv, a plane residual or the tensor-core PSMCosine kernel.  A residual whose fp32 tensor is not valid is read
        from its planes.  res_up=True (fp16-split engine, fp32 residual): `res` has half the output size and is added nearest-upsampled
        (the FPN top-down add).  tiles = (list [cap, 4] int32, count [1] int32, store map [B, H, W] uint8) on the device (`tower_tiles`,
        `tiles_ok` layers): the conv runs on the listed 8 x 16 tiles only and stores the pixels of the map, bit-identical to the dense conv
        there; `out.valid` becomes the map."""
        assert x.C == self.Cin, (x.C, self.Cin)
        assert out.C == self.Cout and out.B == x.B
        Ho, Wo = self.out_hw(x.H, x.W)
        assert (out.H, out.W) == (Ho, Wo), ((out.H, out.W), (Ho, Wo))
        r = self.relu if relu is None else relu
        if tiles is not None and (res_up or not self.tiles_ok()):
            raise _lib.Vd3dError("tile-listed conv: a 3x3 / pad 1 / stride 1 layer of the fp16-split engine without an upsampled residual only")
        if res_up:
            self._check_tc16_input(x, "conv with an upsampled residual")
            if not out.h16 or res is None:
                raise _lib.Vd3dError("conv with an upsampled residual: needs a residual and an output with fp16 (hi, lo) planes")
            need_f32(res, "upsampled conv residual")
            self._tc16([x], [out], [res], True, r, True)
            out.f32, out.lo_fresh = True, True
            return out
        if self.engine != "tc16" or not out.h16 or getattr(self, "passes", 3) != 3:
            f32_out = True
        out.f32 = f32_out
        if self.engine != "tc16" and res is not None:
            need_f32(res, "conv residual")
        if self.engine == "simt":
            need_f32(x, "SIMT conv")
            call("vd3d_conv2d_nhwc", x.ptr, x.B, x.H, x.W, x.C, x.cs, x.co, self.w.data_ptr(), self.b.data_ptr(),
                 self.KH, self.KW, self.stride, self.pad, self.dil,
                 res.ptr if res is not None else None, res.cs if res is not None else 0, res.co if res is not None else 0,
                 out.ptr, self.Cout, out.cs, out.co, 1 if r else 0, _stream())
            return out
        if self.engine == "tc16":
            if not x.h16:
                raise _lib.Vd3dError("fp16-split tensor-core conv: input activation has no fp16 (hi, lo) planes (plan bug: missing split_lo)")
            if CHECK_LO:
                check_lo(x)
            res_planes = res is not None and not res.f32
            if res_planes and self.passes != 3:
                raise _lib.Vd3dError("the 2-pass experiment mode needs VD3D_PLANES=0 (fp32 residuals)")
            if res_planes and not res.h16:
                raise _lib.Vd3dError("conv residual: neither an fp32 tensor nor fp16 planes are valid")
            if tiles is not None:
                self._tc16_tiles(x, out, res, r, f32_out, tiles)
            else:
                self._tc16([x], [out], [res] if res is not None else None, False, r, f32_out)
            out.lo_fresh = out.h16
            out.valid = tiles[2] if tiles is not None else None
            return out
        passes = 3 if self.engine == "tc" else 1
        if passes == 3 and x.lo_ptr is None:
            raise _lib.Vd3dError("tensor-core conv: input activation has no `lo` companion (plan bug: missing split_lo)")
        if CHECK_LO and passes == 3:
            check_lo(x)
        call("vd3d_conv2d_tc", x.ptr, x.lo_ptr, x.B, x.H, x.W, x.C, x.cs, x.co, self.w_hi.data_ptr(), self.w_lo.data_ptr(),
             self.b.data_ptr(), self.KH, self.KW, self.pad, self.dil,
             res.ptr if res is not None else None, res.cs if res is not None else 0, res.co if res is not None else 0,
             out.ptr, out.lo_ptr, self.Cout, out.cs, out.co, 1 if r else 0, passes, self.bn_tile, _stream())
        return out


def fold_bn_transposed(weight, bias, bn: Optional[Dict[str, torch.Tensor]], eps: float = 1e-5):
    """ConvTranspose2d (+bias) followed by eval-mode BatchNorm -> (weight', bias') in float64.  The transposed weight is [Cin, Cout, KH, KW]:
    the BN scale multiplies dim 1 (the output channel), not dim 0 as in `fold_bn`."""
    w, b = fold_bn(weight.detach().transpose(0, 1), bias, bn, eps)
    return w.transpose(0, 1).contiguous(), b


def convtranspose_phase_matrix(w: torch.Tensor, cin_pad: int) -> torch.Tensor:
    """Folded float64 ConvTranspose2d(4, stride 2, padding 1) weight [Cin, Cout, 4, 4] -> the four sub-pixel phase convs as one
    [4 Cout][4 cin_pad] matrix (the weight operand of vd3d_convtranspose2d_tc16): output pixel (2m + r, 2n + s) is the 2x2 conv
    y = sum_{a, c} x[m + r - 1 + a, n + s - 1 + c] . w[:, :, 3 - r - 2a, 3 - s - 2c], so row (2r + s) Cout + co, column (2a + c) cin_pad + ci
    holds w[ci, co, 3 - r - 2a, 3 - s - 2c] (zero for ci >= Cin)."""
    Cin, Cout, KH, KW = w.shape
    assert (KH, KW) == (4, 4) and cin_pad >= Cin
    m = torch.zeros(4, Cout, 4, cin_pad, dtype=torch.float64)
    for r in (0, 1):
        for s in (0, 1):
            for a in (0, 1):
                for c in (0, 1):
                    m[2 * r + s, :, 2 * a + c, :Cin] = w[:, :, 3 - r - 2 * a, 3 - s - 2 * c].t().double()
    return m.reshape(4 * Cout, 4 * cin_pad)


class ConvTransposeLayer:
    """ConvTranspose2d(kernel 4, stride 2, padding 1) + folded eval-mode BatchNorm [+ ReLU] (the CenterNet up-sampling of the ResNet KM3D /
    MonoFlex core, R/detectors/KM3D_core.py:37-47) as its four sub-pixel phase convs in one launch of the fp16-split engine
    (vd3d_convtranspose2d_tc16): 2x2 taps per output pixel.  Runs on that engine only; under any other VD3D_CONV_ENGINE the layer
    refuses to build."""

    def __init__(self, weight, bn=None, bias=None, relu=True, device="cuda"):
        Cin, Cout, KH, KW = weight.shape
        eng = conv_engine_default()
        if eng != "tc16":
            raise _lib.Vd3dError(f"ConvTransposeLayer: the transposed conv runs on the fp16-split tensor-core engine only "
                                 f"(VD3D_CONV_ENGINE=tc16), not {eng!r}")
        if (KH, KW) != (4, 4) or Cin % 8 or Cout % 16:
            raise _lib.Vd3dError(f"ConvTransposeLayer: needs a 4x4 kernel, Cin % 8 == 0 and Cout % 16 == 0 (got {Cin} -> {Cout}, {KH}x{KW})")
        w, b = fold_bn_transposed(weight, bias, bn)
        self.Cin, self.Cout, self.relu = Cin, Cout, relu
        self.engine = "tc16"
        hi, lo, self.out_scale = fp16_split_scaled(convtranspose_phase_matrix(w, (Cin + 63) // 64 * 64))
        self.w_hi, self.w_lo = hi.to(device), lo.to(device)
        self.b = b.float().to(device)
        # 128-column tiles: the widest the engine runs, and the planes-only epilogue keeps its registers there (as the head stem's)
        self.bn_tile = 128 if Cout % 128 == 0 else 0

    @staticmethod
    def out_hw(H, W):
        return 2 * H, 2 * W

    def __call__(self, x: Act, out: Act, f32_out: bool = True):
        """out = relu(bn(conv_transpose(x))) at twice the size of x.  x must carry fresh fp16 (hi, lo) planes; f32_out=False writes the
        output planes only (legal when every consumer is a tensor-core conv)."""
        assert x.C == self.Cin and out.C == self.Cout and out.B == x.B and (out.H, out.W) == self.out_hw(x.H, x.W)
        if not x.h16:
            raise _lib.Vd3dError("transposed conv: input activation has no fp16 (hi, lo) planes (plan bug: missing split_lo)")
        if CHECK_LO:
            check_lo(x)
        if not f32_out and not out.h16:
            raise _lib.Vd3dError("transposed conv: a planes-only output needs an activation with fp16 (hi, lo) planes")
        xh, xl = x.h16_ptrs
        oh, ol = out.h16_ptrs
        call("vd3d_convtranspose2d_tc16", xh, xl, x.B, x.H, x.W, self.Cin, x.cs, x.co, self.w_hi.data_ptr(), self.w_lo.data_ptr(),
             self.out_scale, self.b.data_ptr(), out.ptr if f32_out else None, oh, ol, self.Cout, out.cs, out.co, 1 if self.relu else 0,
             self.bn_tile, _stream())
        out.f32, out.lo_fresh = bool(f32_out), out.h16
        return out


class StemLayer:
    """Few-channel KxK strided stem conv (conv1 7x7 s2 + BN + ReLU, R/backbones/resnet.py:120-122,186-188) on the tensor cores:
    the NCHW image is converted straight into zero-padded fp16 (hi, lo) row planes and the conv runs as a KHx1 convolution
    over 64 virtual channels (see conv2d_tc.cu, vd3d_conv2d_tc16_stem)."""

    def __init__(self, weight, bn=None, stride=2, pad=3, relu=True, device="cuda"):
        w, b = fold_bn(weight, None, bn)
        Cout, Cin, KH, KW = w.shape
        assert Cin <= 4 and KW <= 16 and stride % 2 == 0 and Cout % 16 == 0 and Cout <= 256
        self.Cin, self.Cout, self.KH, self.KW, self.stride, self.pad, self.relu = Cin, Cout, KH, KW, stride, pad, relu
        import os
        self.win = 32 if (KW <= 8 and os.environ.get("VD3D_STEM_WIN", "32") != "64") else 64     # window elements per filter row (8 or 16 pixels x 4)
        wk = torch.zeros(Cout, KH, self.win // 4, 4, dtype=torch.float64)
        wk[:, :, :KW, :Cin] = w.permute(0, 2, 3, 1)
        hi, lo, self.out_scale = fp16_split_scaled(wk.reshape(Cout, KH * self.win))
        self.w_hi, self.w_lo = hi.to(device), lo.to(device)
        self.b = b.float().to(device)

    def out_hw(self, H, W):
        return (H + 2 * self.pad - self.KH) // self.stride + 1, (W + 2 * self.pad - self.KW) // self.stride + 1

    def row_kernel_ok(self) -> bool:
        """the row-strip stem + pool kernel (stem_pool_kernel, csrc/row_conv.cu) covers this layer: 7x7 / 2 / 3, 64 outputs, ReLU, 32-element windows (VD3D_STEM_ROWS=0: off)"""
        import os
        return (self.KH, self.KW, self.stride, self.pad, self.Cout, self.win) == (7, 7, 2, 3, 64, 32) and self.relu and \
            os.environ.get("VD3D_STEM_ROWS", "1") != "0"

    def __call__(self, img_nchw, out: Act, arena: "Arena", name: str, pool: bool = False, f32_out: bool = True):
        """`img_nchw`: one [B, C, H, W] tensor, or a list of such tensors that together form the batch (the stereo plan passes
        [left, right]: each part is converted straight into its batch range of the row planes, no concatenated copy exists)."""
        parts = list(img_nchw) if isinstance(img_nchw, (list, tuple)) else [img_nchw]
        parts = [p.contiguous().float() for p in parts]
        for p in parts:
            _require_cuda(p, "stem")
        _, C, H, W = parts[0].shape
        B = sum(int(p.shape[0]) for p in parts)
        assert all(tuple(p.shape[1:]) == (C, H, W) for p in parts)
        assert C == self.Cin and out.C == self.Cout and out.B == B
        import os
        pool = pool and os.environ.get("VD3D_STEM_POOL", "1") != "0"
        if pool and self.row_kernel_ok() and out.h16:
            # conv + BN + ReLU + MaxPool2d(3, 2, 1) as the row-strip kernel (stem_pool_kernel, csrc/row_conv.cu): `out` is the POOLED tensor, written as fp16 planes
            # (the layer-1 convs and their plane residual read nothing else) and as fp32 only when `f32_out` asks for it
            Hs, Ws = self.out_hw(H, W)
            assert (out.H, out.W) == ((Hs - 1) // 2 + 1, (Ws - 1) // 2 + 1) and out.h16, "fused stem: pooled shape, fp16 planes"
            lib = _lib.load()
            Wp, xoff = int(lib.vd3d_stem_pool_row_pitch(W)), int(lib.vd3d_stem_pool_xoff())
            planes = arena.get(name + ".rows5#h16", (2, B, H, Wp, 4), parts[0].device, dtype=torch.float16, zero=True)   # borders stay zero
            b0 = 0
            for p in parts:
                nb = int(p.shape[0])
                call("vd3d_image_to_h16_rows", p.data_ptr(), nb, C, H, W, planes[0, b0:b0 + nb].data_ptr(), planes[1, b0:b0 + nb].data_ptr(),
                     Wp, xoff, _stream())
                b0 += nb
            oh, ol = out.h16_ptrs
            call("vd3d_stem_pool_fused", planes[0].data_ptr(), planes[1].data_ptr(), B, H, W, Wp, self.w_hi.data_ptr(), self.w_lo.data_ptr(), self.out_scale,
                 self.b.data_ptr(), out.ptr if f32_out else None, oh, ol, out.cs, out.co, _stream())
            out.f32 = bool(f32_out)
            self.wrote_planes = True
            return out
        self.wrote_planes = False
        Wp = int(_lib.load().vd3d_stem_row_pitch(W, self.KW, self.stride, self.pad))
        planes = arena.get(name + ".rows#h16", (2, B, H, Wp, 4), parts[0].device, dtype=torch.float16, zero=True)   # borders stay zero
        b0 = 0
        for p in parts:
            nb = int(p.shape[0])
            call("vd3d_image_to_h16_rows", p.data_ptr(), nb, C, H, W, planes[0, b0:b0 + nb].data_ptr(), planes[1, b0:b0 + nb].data_ptr(),
                 Wp, self.pad, _stream())
            b0 += nb
        if pool:
            # conv + BN + ReLU + MaxPool2d(3, 2, 1) in one kernel: `out` is the POOLED tensor, the conv output is never written
            Hs, Ws = self.out_hw(H, W)
            assert self.relu and self.Cout == 64 and (out.H, out.W) == ((Hs - 1) // 2 + 1, (Ws - 1) // 2 + 1), "fused stem pool: 64 channels, ReLU, pooled shape"
            call("vd3d_conv2d_tc16_stem_pool", planes[0].data_ptr(), planes[1].data_ptr(), B, H, W, Wp, self.KH, self.KW, self.stride, self.pad, self.win,
                 self.w_hi.data_ptr(), self.w_lo.data_ptr(), self.out_scale, self.b.data_ptr(), out.ptr, self.Cout, out.cs, out.co, _stream())
            out.f32 = True
            return out
        oh, ol = out.h16_ptrs
        call("vd3d_conv2d_tc16_stem", planes[0].data_ptr(), planes[1].data_ptr(), B, H, W, Wp, self.KH, self.KW, self.stride, self.pad, self.win,
             self.w_hi.data_ptr(), self.w_lo.data_ptr(), self.out_scale, self.b.data_ptr(), out.ptr, oh, ol, self.Cout, out.cs, out.co,
             1 if self.relu else 0, _stream())
        return out


class RowPlanes:
    """fp16 (hi, lo) ROW PLANES of a few-channel NHWC tensor, the input form of `RowConvLayer`: t = [2, B, H, Wp, PC] (zero outside the image
    columns), image column x at pixel xoff + x of the padded row."""

    def __init__(self, t: torch.Tensor, W: int, xoff: int):
        assert t.dtype == torch.float16 and t.dim() == 5 and t.shape[0] == 2 and t.is_contiguous()
        self.t, self.W, self.xoff = t, int(W), int(xoff)

    B = property(lambda s: s.t.shape[1])
    H = property(lambda s: s.t.shape[2])
    Wp = property(lambda s: s.t.shape[3])
    pc = property(lambda s: s.t.shape[4])


class RowConvLayer:
    """Few-channel KHxKW conv + folded BN [+ ReLU] on the tensor cores as a row-strip kernel (csrc/row_conv.cu): the DLA-34 front end
    (base_layer 7x7 3 -> 16, level0 3x3 16 -> 16, level1 3x3 / 2 16 -> 32, R/networks/backbones/dla.py:246-262), which the generic engine leaves to the
    exact-fp32 SIMT kernel because Cin < 32.  `pc_in` = channels per pixel of the input planes (8 for the image, else Cin)."""

    def __init__(self, weight, bn=None, stride=1, pad=0, relu=True, pc_in: Optional[int] = None, device="cuda"):
        w, b = fold_bn(weight, None, bn)
        Cout, Cin, KH, KW = w.shape
        pc = int(pc_in or Cin)
        assert Cout in (16, 32) and pc in (4, 8, 16) and Cin <= pc and KW * pc * 2 <= 128 and KH <= 7 and stride in (1, 2)
        self.Cin, self.Cout, self.KH, self.KW, self.stride, self.pad, self.relu, self.pc = Cin, Cout, KH, KW, stride, pad, relu, pc
        self.KS = 2 if KW * pc * 2 <= 64 else 4
        wk = torch.zeros(Cout, KH, self.KS * 16, dtype=torch.float64)
        wk[:, :, :KW * pc].view(Cout, KH, KW, pc)[..., :Cin] = w.permute(0, 2, 3, 1)
        hi, lo, self.out_scale = fp16_split_scaled(wk.reshape(Cout, KH * self.KS * 16))
        self.w_hi, self.w_lo = hi.to(device), lo.to(device)
        self.b = b.float().to(device)
        self.engine = "tc16"

    def out_hw(self, H, W):
        return (H + 2 * self.pad - self.KH) // self.stride + 1, (W + 2 * self.pad - self.KW) // self.stride + 1

    def in_pitch(self, W: int, xoff: int) -> int:
        """row pitch (pixels) the INPUT planes of this layer need for W image columns with `xoff` zero pixels in front of every row"""
        v = int(_lib.load().vd3d_row_conv_pitch(W, self.pc, self.KW, self.stride, self.pad, xoff))
        if v <= 0:
            raise _lib.Vd3dError("RowConvLayer: unsupported geometry")
        return v

    def __call__(self, x: RowPlanes, out_planes: Optional[torch.Tensor] = None, out_f32: Optional[torch.Tensor] = None, out_xoff: int = 0, out_co: int = 0):
        """out_planes: [2, B, Ho, out_W, cs] fp16 and / or out_f32: [B, Ho, out_W, cs] fp32 (same out_W / cs); image column x lands at out_xoff + x."""
        assert x.pc == self.pc and (out_planes is not None or out_f32 is not None)
        Ho, Wo = self.out_hw(x.H, x.W)
        ref = out_f32 if out_f32 is not None else out_planes[0]
        assert tuple(ref.shape[:2]) == (x.B, Ho) and ref.shape[2] >= Wo + out_xoff and ref.is_contiguous()
        if out_planes is not None and out_f32 is not None:
            assert tuple(out_planes.shape[1:]) == tuple(out_f32.shape)
        call("vd3d_row_conv", x.t[0].data_ptr(), x.t[1].data_ptr(), x.B, x.H, x.W, x.Wp, x.xoff, self.pc, self.KH, self.KW, self.stride, self.pad,
             self.w_hi.data_ptr(), self.w_lo.data_ptr(), self.out_scale, self.b.data_ptr(), 1 if self.relu else 0, self.Cout,
             out_f32.data_ptr() if out_f32 is not None else None,
             out_planes[0].data_ptr() if out_planes is not None else None, out_planes[1].data_ptr() if out_planes is not None else None,
             int(ref.shape[2]), out_xoff, int(ref.shape[3]), out_co, _stream())
        return Ho, Wo


def image_to_row_planes(img: torch.Tensor, planes: torch.Tensor, xoff: int):
    """NCHW float image -> fp16 (hi, lo) row planes [2, B, H, Wp, 4 | 8] (channels beyond C zero), image column x at xoff + x."""
    _require_cuda(img, "image")
    B, C, H, W = img.shape
    assert planes.dtype == torch.float16 and tuple(planes.shape[:3]) == (2, B, H) and planes.shape[4] in (4, 8) and planes.shape[3] >= W + xoff
    img = img.contiguous().float()
    call("vd3d_image_to_h16_rows_c", img.data_ptr(), B, C, H, W, planes[0].data_ptr(), planes[1].data_ptr(), int(planes.shape[3]), xoff, int(planes.shape[4]), _stream())
    return RowPlanes(planes, W, xoff)


class DeformConvLayer:
    """ModulatedDeformConvPack (R/lib/ops/dcn/deform_conv.py:408-466) [+ folded BN] [+ ReLU] on NHWC activations:
    3x3 offset/mask conv (conv engine) -> deformable im2col with the mask sigmoid fused -> ONE wgmma 1x1 GEMM over
    K = KH*KW*C for the whole batch (the reference loops over images and calls cuBLAS per image)."""

    def __init__(self, weight, bias, off_weight, off_bias, bn=None, stride=1, pad=1, dil=1, deform_groups=1, relu=False, device="cuda"):
        Cout, C, KH, KW = weight.shape
        self.C, self.Cout, self.KH, self.KW = C, Cout, KH, KW
        self.stride, self.pad, self.dil, self.dg = stride, pad, dil, deform_groups
        K = KH * KW
        n_off = 3 * K * deform_groups
        assert off_weight.shape[0] == n_off
        n_pad = (n_off + 15) // 16 * 16                      # tensor-core eligible width (zero filters)
        ow = torch.zeros(n_pad, C, KH, KW, dtype=off_weight.dtype)
        ow[:n_off] = off_weight.detach().cpu()
        ob = torch.zeros(n_pad, dtype=off_weight.dtype)
        ob[:n_off] = off_bias.detach().cpu()
        self.n_off_pad = n_pad
        self.off_conv = ConvLayer(ow, ob, None, stride=stride, pad=pad, dil=dil, relu=False, device=device)   # conv_offset shares stride / padding / dilation (deform_conv.py:441-449)
        # K order of the GEMM: tap-major (k = tap * C + c) in general; 64-channel chunk outermost (k = (chunk * K + tap) * 64 + c % 64) when the
        # staged fused kernel can take the layer (it stages one chunk of the input neighbourhood in shared memory and runs the nine taps on it)
        self.k_order = 1 if (C % 64 == 0 and deform_groups == 1 and KH == 3 and KW == 3 and stride == 1 and pad == 1 and dil == 1
                             and conv_engine_default() == "tc16" and str(device).startswith("cuda")) else 0
        wt = weight.detach().cpu().permute(0, 2, 3, 1).reshape(Cout, K, C)
        if self.k_order:
            wt = wt.reshape(Cout, K, C // 64, 64).permute(0, 2, 1, 3)
        w1 = wt.reshape(Cout, K * C, 1, 1)
        self.main = ConvLayer(w1, bias, bn, relu=relu, device=device)

    def out_hw(self, H, W):
        Ho = (H + 2 * self.pad - (self.dil * (self.KH - 1) + 1)) // self.stride + 1
        Wo = (W + 2 * self.pad - (self.dil * (self.KW - 1) + 1)) // self.stride + 1
        return Ho, Wo

    def __call__(self, x: Act, out: Act, arena: "Arena", name: str, res: Optional[Act] = None):
        """x must carry a fresh lo companion when the offset conv runs on the tensor cores."""
        B, dev = x.B, x.t.device
        Ho, Wo = self.out_hw(x.H, x.W)
        K = self.KH * self.KW
        om = self.off_conv(x, arena.act(name + ".om", (B, Ho, Wo, self.n_off_pad), dev))
        need_f32(x, "deformable gather")
        if self.fused_ok():
            # gather -> shared-memory operand -> wgmma GEMM in ONE kernel: the column tensor never exists (csrc/dcn_fused.cu)
            m = self.main
            oh, ol = out.h16_ptrs
            out.f32 = True
            if res is not None:
                need_f32(res, "deformable conv residual")
            call("vd3d_deform_conv_fused", x.ptr, B, x.H, x.W, x.C, x.cs, x.co, om.ptr, om.cs, 0, 2 * K * self.dg, 1, 1,
                 self.KH, self.KW, self.stride, self.pad, self.dil, self.k_order, m.w_hi.data_ptr(), m.w_lo.data_ptr(), m.out_scale, m.b.data_ptr(),
                 res.ptr if res is not None else None, res.cs if res is not None else 0, res.co if res is not None else 0,
                 out.ptr, oh, ol, m.Cout, out.cs, out.co, 1 if m.relu else 0, _stream())
            out.lo_fresh = oh is not None
            return out
        cols = arena.act("dcn.cols", (B, Ho, Wo, K * self.C), dev, lo=self.main.engine != "simt")     # one buffer per shape, shared by all DCN layers
        if cols.h16:      # the fp16-split GEMM reads only the planes: the gather writes them directly, the fp32 columns are never stored
            ch, cl = cols.h16_ptrs
            call("vd3d_deform_im2col_h16", x.ptr, B, x.H, x.W, x.C, x.cs, x.co, om.ptr, om.cs, 0,
                 om.ptr, om.cs, 2 * K * self.dg, 1, self.KH, self.KW, self.stride, self.pad, self.dil, self.dg, self.k_order,
                 cols.ptr if CHECK_LO else None, ch, cl, cols.cs, _stream())
        else:
            if self.k_order:
                raise _lib.Vd3dError("DeformConvLayer: the chunk-major K order is only produced by the fp16-plane gather (engine tc16)")
            call("vd3d_deform_im2col_nhwc", x.ptr, B, x.H, x.W, x.C, x.cs, x.co, om.ptr, om.cs, 0,
                 om.ptr, om.cs, 2 * K * self.dg, 1, self.KH, self.KW, self.stride, self.pad, self.dil, self.dg,
                 cols.ptr, cols.lo_ptr, cols.cs, _stream())
        return self.main(cols, out, res=res)

    def fused_ok(self) -> bool:
        """the fused gather + GEMM kernel takes this layer (VD3D_DCN_FUSED=0 forces the im2col-planes + 1x1-conv path, kept for A/B and tests)"""
        import os
        return (self.main.engine == "tc16" and os.environ.get("VD3D_DCN_FUSED", "1") != "0" and self.KH * self.KW <= 9 and self.dg == 1 and self.C % 64 == 0)


class DwConvLayer:
    """Depthwise 3x3 (stride 1, pad 1) + folded BN (+ReLU): weights [9][C]."""

    def __init__(self, weight, bn=None, relu=True, device="cuda"):
        w, b = fold_bn(weight, None, bn)          # [C,1,3,3]
        C = w.shape[0]
        assert w.shape[1] == 1 and w.shape[2] == 3 and w.shape[3] == 3
        self.C, self.relu = C, relu
        self.w = w.view(C, 9).t().contiguous().float().to(device)
        self.b = b.float().to(device)

    def __call__(self, x: Act, out: Act):
        assert x.C == self.C and out.C == self.C
        need_f32(x, "dwconv3x3")
        call("vd3d_dwconv3x3_nhwc", x.ptr, x.B, x.H, x.W, x.C, x.cs, x.co, self.w.data_ptr(), self.b.data_ptr(),
             out.ptr, out.cs, out.co, 1 if self.relu else 0, _stream())
        return out


# -------------------------------------------------------------------------------------------------------------
# functional launchers
# -------------------------------------------------------------------------------------------------------------
import os as _os
CHECK_LO = _os.environ.get("VD3D_CHECK_LO", "0") == "1"


def split_lo(x: Act) -> Act:
    """Refresh the `lo` companion of a channel slice written by a non-tensor-core producer."""
    if x.lo is None:
        return x
    need_f32(x, "split_lo")
    if x.h16:
        h, l = x.h16_ptrs
        call("vd3d_split_h16_nhwc", x.ptr, h, l, x.B * x.H * x.W, x.C, x.cs, x.co, _stream())
    else:
        call("vd3d_split_lo_nhwc", x.ptr, x.lo_ptr, x.B * x.H * x.W, x.C, x.cs, x.co, _stream())
    x.lo_fresh = True
    return x


def split_lo_if_stale(x: Act) -> Act:
    """`split_lo` unless the producer of this view wrote the companion itself (`Act.lo_fresh`: set by the fp16-split tensor-core convs, the fused
    deformable conv and the row convs on their OUTPUT view; every other view, slice or later writer starts / stays stale)."""
    if x.lo is None:
        return x
    if x.lo_fresh:
        if CHECK_LO:
            check_lo(x)
        return x
    return split_lo(x)


def check_lo(x: Act):
    """Debug (VD3D_CHECK_LO=1): assert the companion of the slice a tensor-core conv is about to read is fresh (at the pixels its producer
    wrote, `Act.valid`: a tile-listed conv leaves the others stale, and no stored pixel of its consumer reads them)."""
    if not x.f32:
        return                      # planes-only tensor: the planes are the tensor
    t = x.t[..., x.co:x.co + x.C]
    if x.h16:
        hi = t.half()
        lo = (t - hi.float()).half()
        ph, pl = x.lo[0][..., x.co:x.co + x.C], x.lo[1][..., x.co:x.co + x.C]
        if x.valid is not None:
            v = x.valid.bool()
            hi, lo, ph, pl = hi[v], lo[v], ph[v], pl[v]
        if not (torch.equal(ph, hi) and torch.equal(pl, lo)):
            raise _lib.Vd3dError("stale fp16 (hi, lo) planes in front of a tensor-core conv")
        return
    hi = (t.contiguous().view(torch.int32) & -8192).view(torch.float32)
    if not torch.equal(x.lo[..., x.co:x.co + x.C], t - hi):
        raise _lib.Vd3dError("stale `lo` companion in front of a tensor-core conv")


def nchw_to_nhwc(x: torch.Tensor, out: Act):
    _require_cuda(x, "nchw_to_nhwc")
    x = x.contiguous().float()
    B, C, H, W = x.shape
    assert out.C >= C and (out.B, out.H, out.W) == (B, H, W)
    call("vd3d_nchw_to_nhwc", x.data_ptr(), out.ptr, B, C, H, W, out.cs, out.co, _stream())
    return out


def maxpool3x3s2(x: Act, out: Act):
    need_f32(x, "maxpool3x3s2")
    call("vd3d_maxpool3x3s2_nhwc", x.ptr, x.B, x.H, x.W, x.C, x.cs, x.co, out.ptr, out.cs, out.co, _stream())
    return out


def avgpool2(x: Act, out: Act):
    need_f32(x, "avgpool2")
    call("vd3d_avgpool2_nhwc", x.ptr, x.B, x.H, x.W, x.C, x.cs, x.co, out.ptr, out.cs, out.co, _stream())
    return out


def copy_channels(x: Act, out: Act):
    need_f32(x, "copy_channels")
    assert x.C == out.C and x.B * x.H * x.W == out.B * out.H * out.W
    call("vd3d_copy_channels_nhwc", x.ptr, x.B * x.H * x.W, x.C, x.cs, x.co, out.ptr, out.cs, out.co, _stream())
    return out


def psm_cosine(left: Act, right: Act, D: int, out: Act):
    need_f32(left, "psm_cosine (SIMT)"), need_f32(right, "psm_cosine (SIMT)")
    assert (left.cs, left.co, left.C) == (right.cs, right.co, right.C) and out.C == D
    call("vd3d_psm_cosine_nhwc", left.ptr, right.ptr, left.B, left.H, left.W, left.C, left.cs, left.co, D,
         out.ptr, out.cs, out.co, _stream())
    return out


def psm_engine_default() -> str:
    """'tc' = tensor-core PSMCosine on the fp16 (hi, lo) feature planes when they exist (default), 'simt' = fp32 SIMT kernels"""
    import os
    return os.environ.get("VD3D_PSM_ENGINE", "tc")


def psm_tc_eligible(C: int, D: int) -> bool:
    """the tensor-core PSMCosine kernel takes this (channels, disparities) shape: it then reads the fp16 planes only"""
    return psm_engine_default() == "tc" and lo_mode() == "h16" and C % 64 == 0 and D % 4 == 0 and D <= 32


def psm_cosine_stereo(f: Act, B: int, D: int, out: Act, planes_fresh: bool):
    """PSMCosine between the left (batch [0, B)) and right (batch [B, 2B)) halves of one feature tensor.  Uses the tensor-core
    kernel when `f` carries fp16 (hi, lo) planes (refreshing them first if the producer was not a tensor-core conv).
    Returns True if it refreshed the planes of `f`."""
    assert f.B == 2 * B and out.C == D
    if f.h16 and psm_engine_default() == "tc" and f.C % 64 == 0 and D % 4 == 0 and D <= 32:
        if not planes_fresh:
            split_lo(f)
        hi, lo = f.lo[0], f.lo[1]
        call("vd3d_psm_cosine_h16", hi[:B].data_ptr(), lo[:B].data_ptr(), hi[B:].data_ptr(), lo[B:].data_ptr(), B * f.H * f.W, f.W, f.C,
             f.cs, f.co, D, out.ptr, out.cs, out.co, _stream())
        return not planes_fresh
    psm_cosine(f.batch(0, B), f.batch(B, 2 * B), D, out)
    return False


def anchor_mask(anchors: torch.Tensor, means_z: torch.Tensor, P2: torch.Tensor, mask: torch.Tensor,
                y_min=-0.5, y_max=1.8, x_thr=40.0):
    B, N, T = P2.shape[0], anchors.shape[0], means_z.shape[0]
    call("vd3d_anchor_mask", anchors.data_ptr(), means_z.data_ptr(), P2.data_ptr(), B, N, T,
         float(np.float32(y_min)), float(np.float32(y_max)), float(np.float32(x_thr)), mask.data_ptr(), _stream())
    return mask


# Anchors per row group of the gathered regression conv: 8 anchors x 12 regression values = the 96 output columns of one of its N tiles
REG_GROUP_ANCHORS = 8


def reg_candidates(cls_preds: torch.Tensor, mask: torch.Tensor, A: int, ncls: int, score_thr: float, lst: torch.Tensor, counts: torch.Tensor,
                   pixmap: Optional[torch.Tensor] = None):
    """The (image, pixel, anchor group) pairs whose regression values the decoder may read (`vd3d_reg_candidates`): `cls_preds` NHWC [B, H, W, A *
    (ncls + 1)], `mask` [B, P * A] with P = H * W -> `lst` [groups, B * P] int32, `counts` [groups] int32 (device); `pixmap` (optional) [B, P]
    uint8: 1 at the pixels listed in some group, 0 elsewhere."""
    B = cls_preds.shape[0]
    P = cls_preds.numel() // (B * A * (ncls + 1))
    assert lst.dtype == counts.dtype == torch.int32 and lst.shape == (counts.shape[0], B * P) and counts.shape[0] == -(-A // REG_GROUP_ANCHORS)
    assert pixmap is None or (pixmap.dtype == torch.uint8 and pixmap.numel() == B * P and pixmap.is_contiguous())
    call("vd3d_reg_candidates", cls_preds.data_ptr(), mask.data_ptr(), B, P, A, ncls, float(np.float32(score_thr)), REG_GROUP_ANCHORS,
         lst.data_ptr(), counts.data_ptr(), pixmap.data_ptr() if pixmap is not None else None, _stream())


def tower_tile_cap(B: int, H: int, W: int) -> int:
    """entries of one depth's tile list (`tower_tiles`): B * (ceil(H / 8) + 1) * ceil(W / 16)"""
    return B * (-(-H // 8) + 1) * -(-W // 16)


def tower_tiles_fit(H: int, W: int) -> bool:
    """`tower_tiles` takes an H x W map: its two byte maps and tile flags fit the 48 KB of shared memory of its one block per depth"""
    return ((2 * H * W + 15) & ~15) + 4 * (-(-H // 8) + 1) * -(-W // 16) <= 48 * 1024


def tower_tiles(cand: torch.Tensor, smaps: torch.Tensor, tiles: torch.Tensor, counts: torch.Tensor):
    """`vd3d_reg_tower_tiles`: candidate pixel map `cand` [B, H, W] uint8 -> for depth d = 1 .. D, `smaps[d - 1]` [B, H, W] uint8 = the pixels
    within d 3x3 steps of a candidate, `tiles[d - 1]` [cap, 4] int32 = the 8 x 16 tiles (b, y0, x0, 0) that hold them (per image from its first
    such row), `counts[d - 1]` int32 = their number.  On the device, no host synchronisation."""
    B, H, W = cand.shape
    D = smaps.shape[0]
    assert cand.dtype == smaps.dtype == torch.uint8 and tiles.dtype == counts.dtype == torch.int32
    assert tuple(smaps.shape) == (D, B, H, W) and tuple(tiles.shape) == (D, tower_tile_cap(B, H, W), 4) and tuple(counts.shape) == (D,)
    call("vd3d_reg_tower_tiles", cand.data_ptr(), B, H, W, D, smaps.data_ptr(), tiles.data_ptr(), counts.data_ptr(), _stream())


RANGE_MSG = ("an activation left the fp16 range (|v| >= 65520) in front of a tensor-core conv: the fp16-split engine keeps activations "
             "unscaled as fp16 (hi, lo) planes.  Results of this forward are invalid; run with VD3D_CONV_ENGINE=tc (3xTF32) or simt.")


def fp16_range_overflowed(reset: bool = True) -> bool:
    """Read (and by default clear) the device-side fp16-range flag; synchronises the current stream."""
    import ctypes
    v = ctypes.c_int(0)
    call("vd3d_fp16_range_check", ctypes.byref(v), 1 if reset else 0, _stream())
    return bool(v.value)


class DecodeNms:
    """Fixed-capacity decode + NMS outputs for a batch (buffers are reused across calls).  `ws_bytes`: the workspace of the decode that
    fills them (default: this anchor decode + NMS; the CenterNet and RetinaNet decodes pass their own size)."""

    def __init__(self, B: int, cap: int, device, ws_bytes=None):
        self.B, self.cap = B, cap
        if ws_bytes is None:
            ws_bytes = _lib.load().vd3d_decode_nms_workspace(B, cap)
        self.ws = torch.empty(int(ws_bytes), dtype=torch.uint8, device=device)
        self.scores = torch.empty(B, cap, dtype=torch.float32, device=device)
        self.boxes = torch.empty(B, cap, 11, dtype=torch.float32, device=device)
        self.cls = torch.empty(B, cap, dtype=torch.int64, device=device)
        self.anchor = torch.empty(B, cap, dtype=torch.int32, device=device)
        self.count = torch.empty(B, dtype=torch.int32, device=device)
        self.ncand = torch.empty(B, dtype=torch.int32, device=device)

    def run(self, cls_preds, reg_preds, anchors, mean_std, mask, ncls, score_thr, iou_thr, img_w, img_h):
        B, N = cls_preds.shape[0], cls_preds.shape[1]
        T = mean_std.shape[1]
        call("vd3d_decode_nms", cls_preds.data_ptr(), reg_preds.data_ptr(), anchors.data_ptr(), mean_std.data_ptr(),
             mask.data_ptr(), B, N, ncls, T, float(np.float32(score_thr)), float(iou_thr), float(img_w), float(img_h),
             self.cap, self.ws.data_ptr(), self.scores.data_ptr(), self.boxes.data_ptr(), self.cls.data_ptr(),
             self.anchor.data_ptr(), self.count.data_ptr(), self.ncand.data_ptr(), _stream())

    def post_opt(self, P2: torch.Tensor, img_w: float = 1280.0, img_h: float = 288.0, step_r_init: float = 0.4, r_lim: float = 0.01,
                 min_depth: float = 3.0, label: int = 0):
        """`post_optimization` of the anchor heads (R/heads/detection_3d_head.py:294-308 -> R/lib/fast_utils/hill_climbing.py): the yaw of
        every kept row with class `label` deeper than `min_depth` is refined in place by hill climbing, one thread per row, stream-ordered
        after the NMS (no host round trip; the reference reads one `.item()` per box and searches on the CPU).  The hull of the projected
        box is clipped to 1280 x 288 like the reference's hard-coded constants (hill_climbing.py:98-103)."""
        call("vd3d_post_opt", self.boxes.data_ptr(), self.cls.data_ptr(), self.count.data_ptr(), P2.data_ptr(), self.B, self.cap,
             float(img_w), float(img_h), float(step_r_init), float(r_lim), float(min_depth), int(label), _stream())

    def post_forward(self, P2: torch.Tensor, original_P: Optional[torch.Tensor] = None, corners: bool = False):
        """Post-forward geometry of `test_one` (R/pipelines/evaluators.py:112-131) on the kept rows, on the device: back-projected box
        (x, y, z, w, h, l, alpha), rotation theta, 2-D boxes in the pixels of the original frame.  Results stay in fixed-capacity
        buffers (`self.box3d [B, cap, 7]`, `self.theta [B, cap]`, `self.box2d [B, cap, 4]`, optionally `self.corners / self.homo`)."""
        dev = self.scores.device
        if getattr(self, "box3d", None) is None:
            self.box3d = torch.empty(self.B, self.cap, 7, dtype=torch.float32, device=dev)
            self.theta = torch.empty(self.B, self.cap, dtype=torch.float32, device=dev)
            self.box2d = torch.empty(self.B, self.cap, 4, dtype=torch.float32, device=dev)
            self.corners = self.homo = None
        if corners and self.corners is None:
            self.corners = torch.empty(self.B, self.cap, 8, 3, dtype=torch.float32, device=dev)
            self.homo = torch.empty(self.B, self.cap, 8, 3, dtype=torch.float32, device=dev)
        call("vd3d_post_forward", self.boxes.data_ptr(), self.count.data_ptr(), P2.data_ptr(),
             original_P.data_ptr() if original_P is not None else None, self.B, self.cap, self.box3d.data_ptr(), self.theta.data_ptr(),
             self.box2d.data_ptr(), self.corners.data_ptr() if corners else None, self.homo.data_ptr() if corners else None, _stream())
        return self

    def results(self):
        """One D2H read of the counts (the only host sync of the forward), then per-image views."""
        counts = self.count.tolist()
        if fp16_range_overflowed():
            raise _lib.Vd3dError(RANGE_MSG)
        out = []
        for b, k in enumerate(counts):
            if k < 0:
                raise _lib.Vd3dError(f"decode_nms: image {b} has {int(self.ncand[b])} candidates > capacity {self.cap}")
            out.append((self.scores[b, :k], self.boxes[b, :k], self.cls[b, :k]))
        return out
