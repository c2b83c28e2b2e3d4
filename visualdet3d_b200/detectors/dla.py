"""DLA-34 backbone + DLA up-sampling (IDAUp / DLAUp / DLASegUpsample with DCNv2 nodes) on the B200 engine.

Parameter holders reproduce the reference `state_dict` keys (R/backbones/dla.py:40-326, R/backbones/dla_utils.py:42-155);
`DLARunner` / `DLAUpRunner` execute them: every Root concat is a set of channel-slice writes, every `up(proj(x)) + prev` add
is fused into the depthwise transposed-conv kernel, every DeformConv (DCNv2 + BN + ReLU) is one deformable im2col launch +
one wgmma GEMM for the whole batch.
"""
from __future__ import annotations

import math
from typing import List

import numpy as np
import torch
import torch.nn as nn

from .. import engine as E
from .._lib import call
from . import modules as M
from .modules import Holder, seq


# ----------------------------------------------------------------------------------------------------------------
# holders
# ----------------------------------------------------------------------------------------------------------------
class DLABlockP(Holder):
    """BasicBlock of dla.py:40-70 (conv1, bn1, conv2, bn2; residual passed in by the Tree)."""

    def __init__(self, inplanes, planes, stride=1, dilation=1):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 3, stride, dilation, dilation=dilation, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, 3, 1, dilation, dilation=dilation, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.stride = stride


class RootP(Holder):
    """dla.py:154-172."""

    def __init__(self, cin, cout, k, residual):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, k, 1, (k - 1) // 2, bias=False)
        self.bn = nn.BatchNorm2d(cout)
        self.residual = residual


class TreeP(Holder):
    """dla.py:175-230 (attribute order tree1, tree2, root, downsample, project as registered by the reference)."""

    def __init__(self, levels, cin, cout, stride=1, level_root=False, root_dim=0, root_kernel_size=1, dilation=1, root_residual=False):
        super().__init__()
        if root_dim == 0:
            root_dim = 2 * cout
        if level_root:
            root_dim += cin
        if levels == 1:
            self.tree1 = DLABlockP(cin, cout, stride, dilation)
            self.tree2 = DLABlockP(cout, cout, 1, dilation)
            self.root = RootP(root_dim, cout, root_kernel_size, root_residual)
        else:
            self.tree1 = TreeP(levels - 1, cin, cout, stride, root_dim=0, root_kernel_size=root_kernel_size, dilation=dilation,
                               root_residual=root_residual)
            self.tree2 = TreeP(levels - 1, cout, cout, root_dim=root_dim + cout, root_kernel_size=root_kernel_size, dilation=dilation,
                               root_residual=root_residual)
        self.level_root, self.root_dim, self.levels, self.stride = level_root, root_dim, levels, stride
        self.cin, self.cout = cin, cout
        self.downsample = nn.MaxPool2d(stride, stride=stride) if stride > 1 else None
        self.project = seq(nn.Conv2d(cin, cout, 1, 1, bias=False), nn.BatchNorm2d(cout)) if cin != cout else None


class DLAP(Holder):
    """dla.py:233-300; `dlanet(depth=34)` = levels [1,1,1,2,2,1], channels [16,32,64,128,256,512] (:334-337)."""

    def __init__(self, depth=34, out_indices=(-1, 0, 1, 2, 3, 4, 5), pretrained=None, name=None, **_):
        super().__init__()
        if depth != 34:
            raise ValueError("Unsupported model depth on the B200 path: only DLA-34 (the depth every in-scope config uses)")
        if pretrained is not None:
            raise RuntimeError("pretrained DLA weights need a network download (dla.py:327-331); load a checkpoint instead")
        levels, ch = [1, 1, 1, 2, 2, 1], [16, 32, 64, 128, 256, 512]
        self.channels, self.out_indices = ch, tuple(out_indices)
        self.base_layer = seq(nn.Conv2d(3, ch[0], 7, 1, 3, bias=False), nn.BatchNorm2d(ch[0]), nn.ReLU(inplace=True))
        self.level0 = self._conv_level(ch[0], ch[0], levels[0])
        self.level1 = self._conv_level(ch[0], ch[1], levels[1], stride=2)
        self.level2 = TreeP(levels[2], ch[1], ch[2], 2, level_root=False)
        self.level3 = TreeP(levels[3], ch[2], ch[3], 2, level_root=True)
        self.level4 = TreeP(levels[4], ch[3], ch[4], 2, level_root=True)
        self.level5 = TreeP(levels[5], ch[4], ch[5], 2, level_root=True)

    @staticmethod
    def _conv_level(cin, cout, convs, stride=1):
        mods = []
        for i in range(convs):
            mods += [nn.Conv2d(cin, cout, 3, stride if i == 0 else 1, 1, bias=False), nn.BatchNorm2d(cout), nn.ReLU(inplace=True)]
            cin = cout
        return seq(*mods)


class DeformConvP(Holder):
    """dla_utils.py:42-56: actf = (BN, ReLU), conv = ModulatedDeformConvPack(chi, cho, 3, 1, 1)."""

    def __init__(self, chi, cho):
        super().__init__()
        self.actf = seq(nn.BatchNorm2d(cho), nn.ReLU(inplace=True))
        self.conv = M.DCNPackP(chi, cho, 3, 1, 1, 1, 1)


class IDAUpP(Holder):
    """dla_utils.py:59-85."""

    def __init__(self, o, channels, up_f):
        super().__init__()
        self.o, self.n = o, len(channels)
        self.up_f = [int(f) for f in up_f]
        for i in range(1, len(channels)):
            f = int(up_f[i])
            setattr(self, f"proj_{i}", DeformConvP(channels[i], o))
            setattr(self, f"up_{i}", nn.ConvTranspose2d(o, o, f * 2, stride=f, padding=f // 2, output_padding=0, groups=o, bias=False))
            setattr(self, f"node_{i}", DeformConvP(o, o))


class DLAUpP(Holder):
    """dla_utils.py:87-112."""

    def __init__(self, startp, channels, scales):
        super().__init__()
        self.startp = startp
        in_channels = list(channels)
        channels = list(channels)
        scales = np.array(scales, dtype=int)
        self.n = len(channels)
        for i in range(len(channels) - 1):
            j = -i - 2
            setattr(self, f"ida_{i}", IDAUpP(channels[j], in_channels[j:], scales[j:] // scales[j]))
            scales[j + 1:] = scales[j]
            in_channels[j + 1:] = [channels[j] for _ in channels[j + 1:]]


class DLASegUpsampleP(Holder):
    """dla_utils.py:123-155."""

    def __init__(self, input_channels, down_ratio=4, last_level=5, out_channel=0, **_):
        super().__init__()
        assert down_ratio in [2, 4, 8, 16]
        self.first_level, self.last_level = int(np.log2(down_ratio)), last_level
        ch = list(input_channels)
        scales = [2 ** i for i in range(len(ch[self.first_level:]))]
        self.dla_up = DLAUpP(self.first_level, ch[self.first_level:], scales)
        if out_channel == 0:
            out_channel = ch[self.first_level]
        self.out_channel = out_channel
        self.ida_up = IDAUpP(out_channel, ch[self.first_level:self.last_level], [2 ** i for i in range(self.last_level - self.first_level)])


# ----------------------------------------------------------------------------------------------------------------
# runners
# ----------------------------------------------------------------------------------------------------------------
def _tc(layer) -> bool:
    return layer.engine != "simt"


class _BlockRun:
    def __init__(self, blk: DLABlockP, dev):
        self.c1 = E.ConvLayer(blk.conv1.weight, None, E.bn_dict(blk.bn1), stride=blk.stride, pad=1, relu=True, device=dev)
        self.c2 = E.ConvLayer(blk.conv2.weight, None, E.bn_dict(blk.bn2), pad=1, relu=True, device=dev)

    def run(self, x: E.Act, residual: E.Act, out: E.Act, ar: E.Arena, name: str) -> E.Act:
        """x may have a stale lo (refreshed here if needed); `out` gets relu(bn2(conv2(relu(bn1(conv1 x)))) + residual)."""
        B, dev = x.B, x.t.device
        if _tc(self.c1):
            E.split_lo_if_stale(x)
        Ho, Wo = self.c1.out_hw(x.H, x.W)
        t = self.c1(x, ar.act(name + ".t", (B, Ho, Wo, self.c1.Cout), dev, lo=_tc(self.c2)))
        if _tc(self.c2) and not _tc(self.c1):
            E.split_lo(t)
        return self.c2(t, out, res=residual)


class _TreeRun:
    def __init__(self, tree: TreeP, dev):
        self.p = tree
        self.project = (E.ConvLayer(tree.project[0].weight, None, E.bn_dict(tree.project[1]), relu=False, device=dev)
                        if tree.project is not None else None)
        if tree.levels == 1:
            self.t1, self.t2 = _BlockRun(tree.tree1, dev), _BlockRun(tree.tree2, dev)
            k = tree.root.conv.kernel_size[0]
            self.root = E.ConvLayer(tree.root.conv.weight, None, E.bn_dict(tree.root.bn), pad=(k - 1) // 2, relu=True, device=dev)
            self.root_residual = tree.root.residual
        else:
            self.t1, self.t2 = _TreeRun(tree.tree1, dev), _TreeRun(tree.tree2, dev)

    def run(self, x: E.Act, ar: E.Arena, name: str, children: List[E.Act] = None) -> E.Act:
        """Tree.forward (dla.py:216-230).  Returns the tree output (plain; lo stale)."""
        p = self.p
        B, dev = x.B, x.t.device
        children = [] if children is None else list(children)
        if p.stride > 1:
            assert p.stride == 2
            bottom = ar.act(name + ".bottom", (B, x.H // 2, x.W // 2, x.C), dev, lo=True)
            call("vd3d_maxpool2x2s2_nhwc", x.ptr, B, x.H, x.W, x.C, x.cs, x.co, bottom.ptr, bottom.cs, bottom.co, E._stream())
        else:
            bottom = x
        if p.level_root:
            children.append(bottom)
        if p.levels == 1:
            if self.project is not None:
                if _tc(self.project):
                    E.split_lo_if_stale(bottom)
                res = self.project(bottom, ar.act(name + ".res", (B, bottom.H, bottom.W, p.cout), dev))
            else:
                res = bottom
            Ho, Wo = bottom.H, bottom.W
            # root input = cat(x2, x1, *children): x2 and x1 are written straight into their slices
            cat_c = 2 * p.cout + sum(c.C for c in children)
            cat = ar.act(name + ".cat", (B, Ho, Wo, cat_c), dev, lo=True)
            x1 = self.t1.run(x, res, cat.slice(p.cout, p.cout), ar, name + ".b1")
            x2 = self.t2.run(x1, x1, cat.slice(0, p.cout), ar, name + ".b2")
            co = 2 * p.cout
            for ch in children:
                E.copy_channels(ch, cat.slice(co, ch.C))
                co += ch.C
            if _tc(self.root):
                if x1.lo_fresh and x2.lo_fresh:       # both block outputs came from tensor-core convs: only the copied children lack their planes
                    if co > 2 * p.cout:
                        E.split_lo(cat.slice(2 * p.cout, co - 2 * p.cout))
                else:
                    E.split_lo(cat)
            out = ar.act(name + ".out", (B, Ho, Wo, p.cout), dev, lo=True)
            return self.root(cat, out, res=x2 if self.root_residual else None)
        # levels > 1: the reference also evaluates project(bottom) here but never uses it (Tree.forward overwrites `residual`)
        x1 = self.t1.run(x, ar, name + ".t1")
        children.append(x1)
        return self.t2.run(x1, ar, name + ".t2", children=children)


class DLARunner:
    """DLA.forward (dla.py:317-326): returns the list of level outputs selected by out_indices (plain Acts, lo stale)."""

    def __init__(self, p: DLAP, dev, first_used_level: int = 0):
        """first_used_level: lowest level output the caller reads (DLASegUpsample: first_level); levels below it need not exist as activations"""
        self.p = p
        self.base = E.ConvLayer(p.base_layer[0].weight, None, E.bn_dict(p.base_layer[1]), pad=3, relu=True, device=dev, cin_pad=4)
        self.l0 = E.ConvLayer(p.level0[0].weight, None, E.bn_dict(p.level0[1]), pad=1, relu=True, device=dev)
        self.l1 = E.ConvLayer(p.level1[0].weight, None, E.bn_dict(p.level1[1]), stride=2, pad=1, relu=True, device=dev)
        self.trees = [_TreeRun(getattr(p, f"level{i}"), dev) for i in range(2, 6)]
        # the three full-resolution layers (Cin < 32: exact-fp32 SIMT kernel in the generic engine, 2.8 ms of a 13 ms MonoFlex step at 384x1280) as
        # row-strip tensor-core kernels on fp16 row planes (csrc/row_conv.cu); VD3D_ROWCONV=0 restores the SIMT path
        import os
        self.rc = None
        if (E.conv_engine_default() == "tc16" and os.environ.get("VD3D_ROWCONV", "1") != "0" and -1 not in p.out_indices and first_used_level >= 2
                and tuple(p.base_layer[0].weight.shape) == (16, 3, 7, 7) and tuple(p.level0[0].weight.shape) == (16, 16, 3, 3)
                and tuple(p.level1[0].weight.shape) == (32, 16, 3, 3)):
            self.rc = (E.RowConvLayer(p.base_layer[0].weight, E.bn_dict(p.base_layer[1]), stride=1, pad=3, relu=True, pc_in=8, device=dev),
                       E.RowConvLayer(p.level0[0].weight, E.bn_dict(p.level0[1]), stride=1, pad=1, relu=True, pc_in=16, device=dev),
                       E.RowConvLayer(p.level1[0].weight, E.bn_dict(p.level1[1]), stride=2, pad=1, relu=True, pc_in=16, device=dev))

    def _front_rows(self, img: torch.Tensor, ar: E.Arena, tag: str) -> E.Act:
        """base_layer -> level0 -> level1 on row planes: image -> 8-channel planes -> 16-channel planes (written straight into the zero-bordered
        input form of the next layer) -> the ordinary NHWC activation (fp32 + planes) of level1"""
        base, l0, l1 = self.rc
        dev = img.device
        B, _, H, W = img.shape
        f16 = torch.float16
        p0 = E.image_to_row_planes(img, ar.get(tag + ".img#rows", (2, B, H, base.in_pitch(W, 4), 8), dev, dtype=f16, zero=True), 4)
        r1 = ar.get(tag + ".base#rows", (2, B, H, l0.in_pitch(W, 2), 16), dev, dtype=f16, zero=True)
        base(p0, r1, None, out_xoff=2)
        r2 = ar.get(tag + ".l0#rows", (2, B, H, l1.in_pitch(W, 2), 16), dev, dtype=f16, zero=True)
        l0(E.RowPlanes(r1, W, 2), r2, None, out_xoff=2)
        H1, W1 = l1.out_hw(H, W)
        x = ar.act(tag + ".l1", (B, H1, W1, 32), dev, lo=True)
        assert x.h16
        l1(E.RowPlanes(r2, W, 2), x.lo, x.t)
        x.lo_fresh = True
        return x

    def run(self, img: torch.Tensor, ar: E.Arena, tag: str = "dla") -> List[E.Act]:
        dev = img.device
        B, _, H, W = img.shape
        if self.rc is not None and ar.lo_form == "h16":
            x = self._front_rows(img, ar, tag)
            # level 0 / 1 outputs exist only as row planes: DLAUp starts at first_level >= 2 (dla_utils.py:106-112) and never reads them; their list
            # slots (the up-sampling path indexes the list by level) hold None
            ys = [None for i in (0, 1) if i in self.p.out_indices]
            for i, tr in enumerate(self.trees):
                x = tr.run(x, ar, f"{tag}.lv{i + 2}")
                if i + 2 in self.p.out_indices:
                    ys.append(x)
            return ys
        x0 = ar.act(tag + ".in4", (B, H, W, 4), dev, zero=True)
        E.nchw_to_nhwc(img, x0)
        ys = []
        x = self.base(x0, ar.act(tag + ".base", (B, H, W, 16), dev, lo=_tc(self.l0)))
        if -1 in self.p.out_indices:
            ys.append(x)
        if _tc(self.l0) and not _tc(self.base):
            E.split_lo(x)
        x = self.l0(x, ar.act(tag + ".l0", (B, H, W, 16), dev, lo=_tc(self.l1)))
        if 0 in self.p.out_indices:
            ys.append(x)
        if _tc(self.l1) and not _tc(self.l0):
            E.split_lo(x)
        x = self.l1(x, ar.act(tag + ".l1", (B, H // 2, W // 2, 32), dev, lo=True))
        if 1 in self.p.out_indices:
            ys.append(x)
        for i, tr in enumerate(self.trees):
            x = tr.run(x, ar, f"{tag}.lv{i + 2}")
            if i + 2 in self.p.out_indices:
                ys.append(x)
        return ys


class _DeformRun:
    def __init__(self, p: DeformConvP, dev):
        c = p.conv
        self.layer = E.DeformConvLayer(c.weight, c.bias, c.conv_offset.weight, c.conv_offset.bias, E.bn_dict(p.actf[0]), c.stride, c.padding,
                                       c.dilation, c.deformable_groups, relu=True, device=dev)

    def run(self, x: E.Act, out: E.Act, ar: E.Arena, name: str) -> E.Act:
        if _tc(self.layer.off_conv):
            E.split_lo_if_stale(x)
        return self.layer(x, out, ar, name)


class _IDAUpRun:
    def __init__(self, p: IDAUpP, dev):
        self.p = p
        self.proj, self.node, self.up_w, self.f = {}, {}, {}, {}
        for i in range(1, p.n):
            self.proj[i] = _DeformRun(getattr(p, f"proj_{i}"), dev)
            self.node[i] = _DeformRun(getattr(p, f"node_{i}"), dev)
            w = getattr(p, f"up_{i}").weight.detach()               # [o, 1, 2f, 2f]
            k = w.shape[-1]
            self.up_w[i] = w.reshape(p.o, k * k).t().contiguous().float().to(dev)      # [k*k][o] tap-major
            self.f[i] = k // 2

    def run(self, layers: List[E.Act], startp: int, endp: int, ar: E.Arena, name: str):
        """IDAUp.forward (dla_utils.py:79-85): layers[i] = node(up(proj(layers[i])) + layers[i-1]), in place in the list."""
        o = self.p.o
        for i in range(startp + 1, endp):
            k = i - startp
            x = layers[i]
            B, dev = x.B, x.t.device
            pr = self.proj[k].run(x, ar.act(f"{name}.p{k}", (B, x.H, x.W, o), dev), ar, f"{name}.p{k}")
            f = self.f[k]
            up = ar.act(f"{name}.u{k}", (B, x.H * f, x.W * f, o), dev, lo=True)
            prev = layers[i - 1]
            assert (prev.H, prev.W, prev.C) == (up.H, up.W, o), ((prev.H, prev.W, prev.C), (up.H, up.W, o))
            call("vd3d_dw_convtranspose_nhwc", pr.ptr, B, pr.H, pr.W, o, pr.cs, pr.co, self.up_w[k].data_ptr(), f,
                 prev.ptr, prev.cs, prev.co, up.ptr, up.cs, up.co, E._stream())
            layers[i] = self.node[k].run(up, ar.act(f"{name}.n{k}", (B, up.H, up.W, o), dev, lo=True), ar, f"{name}.n{k}")


class DLAUpRunner:
    """DLASegUpsample.forward (dla_utils.py:147-155) = DLAUp.forward (:106-112) + the final IDAUp."""

    def __init__(self, p: DLASegUpsampleP, dev):
        self.p = p
        self.idas = [_IDAUpRun(getattr(p.dla_up, f"ida_{i}"), dev) for i in range(p.dla_up.n - 1)]
        self.final = _IDAUpRun(p.ida_up, dev)

    def run(self, tensors: List[E.Act], ar: E.Arena, tag: str = "up") -> E.Act:
        layers = list(tensors)
        startp = self.p.dla_up.startp
        out = [layers[-1]]
        for i in range(len(layers) - startp - 1):
            self.idas[i].run(layers, len(layers) - i - 2, len(layers), ar, f"{tag}.ida{i}")
            out.insert(0, layers[-1])
        y = [out[i] for i in range(self.p.last_level - self.p.first_level)]
        self.final.run(y, 0, len(y), ar, f"{tag}.fin")
        return y[-1]
