"""Host-side weight preparation of the conv engine (no GPU): BN folding in float64, the fp16 (hi, lo) split and the power-of-two weight
scaling that keeps the lo parts normal, the stem's row-window weight layout."""
import numpy as np
import torch
import torch.nn.functional as F

from visualdet3d_b200 import engine as E


def test_fold_bn_equals_conv_then_bn():
    g = torch.Generator().manual_seed(0)
    w = torch.randn(12, 5, 3, 3, generator=g, dtype=torch.float64)
    b = torch.randn(12, generator=g, dtype=torch.float64)
    bn = dict(weight=torch.rand(12, generator=g, dtype=torch.float64) + 0.5, bias=torch.randn(12, generator=g, dtype=torch.float64),
              running_mean=torch.randn(12, generator=g, dtype=torch.float64), running_var=torch.rand(12, generator=g, dtype=torch.float64) + 0.1)
    x = torch.randn(2, 5, 9, 11, generator=g, dtype=torch.float64)
    ref = F.batch_norm(F.conv2d(x, w, b, padding=1), bn["running_mean"], bn["running_var"], bn["weight"], bn["bias"], False, 0.0, 1e-5)
    wf, bf = E.fold_bn(w, b, bn)
    got = F.conv2d(x, wf, bf, padding=1)
    assert float((got - ref).abs().max()) < 1e-12
    wf2, bf2 = E.fold_bn(w, None, None)
    assert torch.equal(wf2, w) and float(bf2.abs().max()) == 0.0


def test_fp16_split_carries_22_bits():
    """hi + lo reproduces v to 2^-22 |v| wherever lo is a normal fp16 number (|v| >= 2^-3), and to half the fp16 subnormal spacing
    (2^-25, absolute) below: activations are not scaled, weights are (next test)."""
    g = torch.Generator().manual_seed(1)
    v = torch.randn(100000, generator=g) * torch.logspace(-3, 3, 100000)
    v = v.clamp(-6e4, 6e4)
    hi, lo = E.fp16_split(v)
    assert hi.dtype == torch.float16 and lo.dtype == torch.float16
    err = (hi.double() + lo.double() - v.double()).abs()
    bound = torch.maximum(v.double().abs() * 2.0 ** -22, torch.full_like(err, 2.0 ** -25))
    assert bool((err <= bound).all())
    assert torch.equal(hi, v.half()) and torch.equal(lo, (v - hi.float()).half())


def test_conv_layer_scales_weights_into_fp16_range():
    """the tensor-core layers store W * 2^k with max |W| 2^k in [8192, 16384) (k within +-24) and undo it with out_scale = 2^-k (exact)"""
    g = torch.Generator().manual_seed(2)
    for scale in (1e-4, 1.0, 300.0):
        w = torch.randn(32, 64, 3, 3, generator=g) * scale
        wm = w.double().reshape(32, -1)
        hi, lo, out_scale = E.fp16_split_scaled(wm)
        wk = wm.abs().max()
        k = int(np.floor(np.log2(16384.0 / float(wk))))
        assert 8192.0 <= float(wk) * 2.0 ** k < 16384.0
        k = max(-24, min(24, k))
        assert out_scale == 2.0 ** -k
        assert all(torch.equal(a, b) for a, b in zip((hi, lo), E.fp16_split(wm * 2.0 ** k)))
        rec = (hi.double() + lo.double()) * out_scale
        assert float((rec - wm).abs().max()) <= float(wk) * 2.0 ** -21
        layer = E.ConvLayer(w, None, None, pad=1, device="cpu", engine="tc16")
        assert layer.engine == "simt"                 # and a CPU-device layer never claims the tensor-core engine
    # the scale stays within 2^+-24, and an all-zero matrix is not scaled
    assert E.fp16_split_scaled(torch.full((4, 8), 1e-12, dtype=torch.float64))[2] == 2.0 ** -24
    assert E.fp16_split_scaled(torch.full((4, 8), 1e12, dtype=torch.float64))[2] == 2.0 ** 24
    assert E.fp16_split_scaled(torch.zeros(4, 8, dtype=torch.float64))[2] == 1.0


def test_stem_weight_layout():
    g = torch.Generator().manual_seed(3)
    w = torch.randn(64, 3, 7, 7, generator=g)
    for win_env, win in (("32", 32), ("64", 64)):
        import os
        os.environ["VD3D_STEM_WIN"] = win_env
        try:
            layer = E.StemLayer(w, None, stride=2, pad=3, relu=True, device="cpu")
        finally:
            os.environ.pop("VD3D_STEM_WIN")
        assert layer.win == win and tuple(layer.w_hi.shape) == (64, 7 * win)
        rec = ((layer.w_hi.double() + layer.w_lo.double()) * layer.out_scale).view(64, 7, win // 4, 4)
        assert float((rec[:, :, :7, :3] - w.permute(0, 2, 3, 1).double()).abs().max()) < float(w.abs().max()) * 2.0 ** -20
        assert float(rec[:, :, 7:, :].abs().max()) == 0.0 and float(rec[:, :, :, 3].abs().max()) == 0.0      # zero beyond KW pixels / 3 channels
        assert layer.out_hw(384, 1280) == (192, 640)


def test_dcn_weight_cache_is_keyed_on_the_tensor_object():
    """ops.dcn packs tensor-core weights once per weight tensor.  The cache must never serve an entry to ANOTHER tensor that happens to
    live at the same address with the same shape and version (a freed model followed by a new one): entries are keyed on the object and
    die with it; in-place updates re-pack."""
    import gc
    from visualdet3d_b200.ops import dcn
    c = dcn._WeightCache()
    g = torch.Generator().manual_seed(0)
    w = torch.randn(8, 4, 3, 3, generator=g)
    h1, l1 = c.get(w)
    assert c.get(w)[0] is h1 and len(c) == 1
    want = w.permute(0, 2, 3, 1).reshape(8, 36).clone()
    assert float((h1 + l1 - want).abs().max()) < 4e-6               # tf32 (hi, lo): 21 significant bits
    w.mul_(2.0)                                            # in-place change -> re-packed
    h2, l2 = c.get(w)
    assert h2 is not h1 and float((h2 + l2 - 2 * want).abs().max()) < 8e-6
    ptr = w.data_ptr()
    del w
    gc.collect()
    assert len(c) == 0                                     # the entry died with its tensor
    # a different tensor, same shape / version / (very likely) the same address: gets its own packing
    w2 = torch.randn(8, 4, 3, 3, generator=g)
    h3, l3 = c.get(w2)
    assert float((h3 + l3 - w2.permute(0, 2, 3, 1).reshape(8, 36)).abs().max()) < 4e-6
    print("same address reused:", w2.data_ptr() == ptr)


def test_anchor_config_is_honoured_or_refused(tmp_path):
    """Every argument the reference's Anchors / head take (R/heads/anchors.py:11-14, detection_3d_head.py:30) is either honoured
    (filter thresholds) or refused loudly (prior channels != 6, read_precompute_anchor=False) -- never silently ignored."""
    import pytest
    from visualdet3d_b200 import synth
    from visualdet3d_b200.detectors import Stereo3D
    obj_types = ["Car", "Pedestrian"]
    pm, ps = synth.synth_priors(16, 3, obj_types)
    synth.write_priors(str(tmp_path), pm, ps, obj_types)
    cfg = synth.stereo3d_cfg(str(tmp_path), obj_types)
    assert Stereo3D(cfg).anchor_filter == (-0.5, 1.8, 40.0)
    cfg["head"]["anchors_cfg"]["filter_y_threshold_min_max"] = (-0.3, 1.5)
    cfg["head"]["anchors_cfg"]["filter_x_threshold"] = 30.0
    assert Stereo3D(cfg).anchor_filter == (-0.3, 1.5, 30.0)
    cfg["head"]["anchors_cfg"]["anchor_prior_channel"] = 7
    with pytest.raises(ValueError):
        Stereo3D(cfg)
    cfg["head"]["anchors_cfg"]["anchor_prior_channel"] = 6
    cfg["head"]["read_precompute_anchor"] = False
    with pytest.raises(ValueError):
        Stereo3D(cfg)


def test_act_views_and_freshness_flag():
    """engine.Act bookkeeping runs without a GPU: slices are new views that start stale (`lo_fresh` False) whatever the parent's state"""
    import torch
    from visualdet3d_b200 import engine as E
    t = torch.zeros(2, 3, 4, 16)
    a = E.Act(t, 0, None, torch.zeros(2, 2, 3, 4, 16, dtype=torch.float16))
    assert a.h16 and a.f32 and not a.lo_fresh and (a.B, a.H, a.W, a.C, a.cs) == (2, 3, 4, 16, 16)
    a.lo_fresh = True
    s = a.slice(8, 8)
    assert (s.co, s.C) == (8, 8) and s.lo is a.lo and not s.lo_fresh
    rp = E.RowPlanes(torch.zeros(2, 1, 4, 12, 8, dtype=torch.float16), W=8, xoff=4)
    assert (rp.B, rp.H, rp.Wp, rp.pc) == (1, 4, 12, 8)
