"""The float64 deformable-convolution restatement of tests/dcn_cases.py and its offset families, checked without a GPU:
  * every family builder hits its targets exactly in float32;
  * the forward equals torchvision's float64 deform_conv2d on every family (torchvision is handed the same float32-rounded positions);
  * the backward equals torchvision's everywhere except d/dh (d/dw) where the position is exactly -1: the reference drops that tap, torchvision
    keeps it.  The difference is asserted to be confined to exactly those entries, with the restatement zero there;
  * the backward matches central finite differences at interior, non-integer positions."""
import numpy as np
import pytest
import torch

import dcn_cases as dc

# B, C, H, W, Cout, KH, stride, pad, dil, dg
SHAPES = [(2, 8, 7, 9, 5, 3, 1, 1, 1, 1), (1, 8, 6, 5, 3, 3, 2, 1, 2, 2), (1, 4, 5, 7, 2, 5, 1, 2, 1, 1), (2, 4, 3, 5, 3, 1, 1, 0, 1, 1)]


def _inputs(shape, family, seed=0):
    B, C, H, W, Co, k, s, p, d, dg = shape
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(Co, C, k, k, generator=g, dtype=torch.float64)
    b = torch.randn(Co, generator=g, dtype=torch.float64)
    off, logit = dc.family_offsets(family, B, H, W, k, k, s, p, d, dg, seed)
    return x, w, b, off, dc.sigmoid_f32(logit).double()


def _tv(x, off_eff, mask, w, b, s, p, d):
    from torchvision.ops import deform_conv2d          # imported where used, like the rest of the suite
    return deform_conv2d(x, off_eff, w, b, stride=s, padding=p, dilation=d, mask=mask)


@pytest.mark.parametrize("family", dc.FAMILIES)
@pytest.mark.parametrize("shape", SHAPES)
def test_family_targets_exact_in_float32(shape, family):
    B, C, H, W, Co, k, s, p, d, dg = shape
    off, logit = dc.family_offsets(family, B, H, W, k, k, s, p, d, dg)
    Ho, Wo = dc.out_hw(H, W, k, k, s, p, d)
    assert off.dtype == torch.float32 and off.shape == (B, 2 * k * k * dg, Ho, Wo) and logit.shape == (B, k * k * dg, Ho, Wo)
    h, w = dc.positions(off, k, k, s, p, d, dg)
    hx, wx = dc.positions(off, k, k, s, p, d, dg, exact=True)
    if family in ("zero", "integer", "half", "knife", "far"):
        assert torch.equal(h, hx) and torch.equal(w, wx)             # base + offset is exact in float32
    frac = lambda t: t - torch.floor(t)
    if family in ("zero", "integer"):
        assert torch.equal(frac(h), torch.zeros_like(h)) and torch.equal(frac(w), torch.zeros_like(w))
    if family == "half":
        assert torch.equal(frac(h), torch.full_like(h, 0.5)) and torch.equal(frac(w), torch.full_like(w, 0.5))
    if family == "knife":
        targets = lambda n: {-1.0, -1.0 + dc.KNIFE_EPS, n - 1.0, n - dc.KNIFE_EPS, float(n)}
        hs, ws = set(h.unique().tolist()), set(w.unique().tolist())
        assert targets(H) <= hs and targets(W) <= ws
        assert all(v in targets(H) or (v == int(v) and 0 <= v <= H - 1) for v in hs)
    if family == "far":
        assert bool(((h <= -1) | (h >= H) | (w <= -1) | (w >= W)).float().mean() > 0.5)
    if family == "mask_extreme":
        m = dc.sigmoid_f32(logit)
        assert set(m.unique().tolist()) <= {0.0, 1.0, float(np.float32(1 / (1 + np.exp(20.0)))), float(np.float32(1 / (1 + np.exp(-20.0))))}
        assert float(dc.sigmoid_f32(torch.tensor([-90.0]))) == 0.0 and float(dc.sigmoid_f32(torch.tensor([90.0]))) == 1.0


def test_boundary_offsets_are_all_invalid():
    for B, H, W, k, s, p, d, dg in ((1, 5, 7, 3, 1, 1, 1, 1), (2, 3, 5, 7, 2, 3, 1, 2)):
        off = dc.boundary_offsets(B, H, W, k, k, s, p, d, dg)
        h, w = dc.positions(off, k, k, s, p, d, dg)
        assert not bool(((h > -1) & (w > -1) & (h < H) & (w < W)).any())
        assert bool(((h == -1) & (w > -1) & (w < W)).any()) and bool(((w == -1) & (h > -1) & (h < H)).any())


@pytest.mark.parametrize("family", dc.FAMILIES)
@pytest.mark.parametrize("shape", SHAPES)
def test_forward_matches_torchvision(shape, family):
    B, C, H, W, Co, k, s, p, d, dg = shape
    x, w, b, off, mask = _inputs(shape, family)
    eff = dc.effective_offsets(off, k, k, s, p, d, dg)
    for m in (mask, None):
        r = dc.forward(x, off, m, w, b, s, p, d, dg)
        want = _tv(x, eff, m, w, b, s, p, d)
        err = float((r["out"] - want).abs().max())
        assert err <= 1e-12 * (1.0 + float(r["abs_out"].max())), (family, err)
        assert bool((r["abs_out"] + 1e-12 >= r["out"].abs()).all())
    # the columns alone: an identity weight over (tap, channel) turns the forward into the column tensor
    Ho, Wo = dc.out_hw(H, W, k, k, s, p, d)
    eye = torch.eye(k * k * C, dtype=torch.float64).reshape(k * k * C, k * k, C).permute(0, 2, 1).reshape(k * k * C, C, k, k)
    want = _tv(x, eff, mask, eye, None, s, p, d).permute(0, 2, 3, 1)
    assert r["cols"].shape == (B, Ho, Wo, k * k * C)
    assert float((dc.forward(x, off, mask, w, b, s, p, d, dg)["cols"] - want).abs().max()) <= 1e-12 * (1.0 + float(want.abs().max()))


@pytest.mark.parametrize("family", dc.FAMILIES)
@pytest.mark.parametrize("shape", SHAPES)
def test_backward_matches_torchvision_except_at_minus_one(shape, family):
    B, C, H, W, Co, k, s, p, d, dg = shape
    x, w, b, off, mask = _inputs(shape, family, seed=1)
    Ho, Wo = dc.out_hw(H, W, k, k, s, p, d)
    gout = torch.randn(B, Co, Ho, Wo, generator=torch.Generator().manual_seed(7), dtype=torch.float64)
    eff = dc.effective_offsets(off, k, k, s, p, d, dg)
    for v2 in (True, False):
        xt, ot, wt, bt = x.clone().requires_grad_(), eff.clone().requires_grad_(), w.clone().requires_grad_(), b.clone().requires_grad_()
        mt = mask.clone().requires_grad_() if v2 else None
        (_tv(xt, ot, mt, wt, bt, s, p, d) * gout).sum().backward()
        r = dc.backward(x, off, mask if v2 else None, w, gout, s, p, d, dg)
        pairs = [("grad_input", xt.grad), ("grad_weight", wt.grad), ("grad_bias", bt.grad)] + ([("grad_mask", mt.grad)] if v2 else [])
        for name, want in pairs:
            err = float((r[name] - want).abs().max())
            assert err <= 1e-12 * (1.0 + float(r["abs_" + name].max())), (name, family, err)
        edge = r["edge"]
        diff = (r["grad_offset"] - ot.grad).abs() > 1e-12 * (1.0 + float(r["abs_grad_offset"].max()))
        assert not bool((diff & ~edge).any()), (family, "grad_offset differs away from the -1 knife edge")
        assert bool((r["grad_offset"][edge] == 0.0).all())             # the reference's rule: no coordinate gradient at exactly -1
        if family == "knife" or (family == "zero" and p > 0):          # both put taps at exactly -1 with a valid other coordinate
            assert bool(edge.any()) and bool(diff.any()) and bool((ot.grad[edge] != 0).any()), "torchvision keeps the tap at -1"


def test_backward_matches_finite_differences():
    """Central differences of L = sum(gout * out) at interior positions whose fractions stay in [0.2, 0.8] under the perturbation (the
    bilinear form is linear along each coordinate inside a cell, so the differences are exact up to rounding)."""
    B, C, H, W, Co, k, s, p, d, dg = 1, 4, 6, 7, 3, 3, 1, 1, 1, 2
    g = torch.Generator().manual_seed(3)
    Ho, Wo = dc.out_hw(H, W, k, k, s, p, d)
    x = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(Co, C, k, k, generator=g, dtype=torch.float64)
    b = torch.randn(Co, generator=g, dtype=torch.float64)
    mask = torch.rand(B, k * k * dg, Ho, Wo, generator=g, dtype=torch.float64) + 0.1
    # positions: a random interior cell (so every corner is inside) plus a fraction in [0.2, 0.8]
    bh, bw = dc.base_positions(Ho, Wo, k, k, s, p, d)
    K = k * k
    ch = torch.randint(0, H - 1, (B, dg, K, Ho, Wo), generator=g).double() + 0.2 + 0.6 * torch.rand(B, dg, K, Ho, Wo, generator=g, dtype=torch.float64)
    cw = torch.randint(0, W - 1, (B, dg, K, Ho, Wo), generator=g).double() + 0.2 + 0.6 * torch.rand(B, dg, K, Ho, Wo, generator=g, dtype=torch.float64)
    off = torch.stack([ch - bh[None, None, :, :, None].double(), cw - bw[None, None, :, None, :].double()], 3).reshape(B, 2 * K * dg, Ho, Wo)
    gout = torch.randn(B, Co, Ho, Wo, generator=g, dtype=torch.float64)
    loss = lambda x_, o_, m_, w_, b_: float((dc.forward(x_, o_, m_, w_, b_, s, p, d, dg, exact=True)["out"] * gout).sum())
    r = dc.backward(x, off, mask, w, gout, s, p, d, dg, exact=True)
    args = dict(x=x, off=off, mask=mask, w=w, b=b)
    names = dict(x="grad_input", off="grad_offset", mask="grad_mask", w="grad_weight", b="grad_bias")
    eps = 1e-6
    for key, gname in names.items():
        t = args[key]
        for i in torch.randperm(t.numel(), generator=g)[:12].tolist():
            plus, minus = dict(args), dict(args)
            tp, tm = t.clone(), t.clone()
            tp.view(-1)[i] += eps
            tm.view(-1)[i] -= eps
            plus[key], minus[key] = tp, tm
            fd = (loss(plus["x"], plus["off"], plus["mask"], plus["w"], plus["b"]) - loss(minus["x"], minus["off"], minus["mask"], minus["w"], minus["b"])) / (2 * eps)
            an = float(r[gname].reshape(-1)[i])
            assert abs(fd - an) <= 1e-6 * (1.0 + abs(an)), (gname, i, fd, an)
