"""CPU-side checks of the drop-in boundary: the C-ABI library loads and exports every symbol the header declares,
the registry mirrors the reference contract, and the detector's state_dict keys equal the reference's."""
import json
import os

import pytest
import torch

from conftest import GOLDEN, ROOT


def test_library_exports_every_declared_symbol():
    from visualdet3d_b200 import _lib
    lib = _lib.load()
    syms = _lib.header_symbols()
    assert len(syms) >= 15
    for s in syms:
        assert hasattr(lib, s), s
    assert lib.vd3d_version() >= 100


def test_registry_contract():
    from visualdet3d_b200.plugin import Registry
    r = Registry("detectors")

    @r.register_module
    class Foo:  # noqa
        pass

    assert r["Foo"] is Foo and r.get("Bar") is None
    with pytest.raises(KeyError):
        r["Bar"]
    with pytest.raises(KeyError):
        r._register_module(Foo)
    r._register_module(Foo, force=True)
    with pytest.raises(TypeError):
        r._register_module(3)
    assert "Foo" in repr(r)


def test_stereo3d_registered_and_state_dict_keys_match_reference():
    from visualdet3d_b200.plugin import DETECTOR_DICT
    from visualdet3d_b200.detectors import build_synthetic_stereo3d
    assert "Stereo3D" in DETECTOR_DICT
    det, sd, cfg, _ = build_synthetic_stereo3d()
    ref = json.load(open(os.path.join(GOLDEN, "stereo3d_keys.json")))
    mine = {k: list(v.shape) for k, v in det.state_dict().items()}
    assert list(mine.keys()) == list(ref.keys())        # same names, same order
    assert mine == ref                                  # same shapes
    assert sum(p.numel() for p in det.parameters()) == sum(
        int(torch.tensor(v).prod()) for k, v in ref.items()
        if not any(t in k for t in ("running_", "num_batches", "balance_weights", "regression_weight")))


def test_product_path_has_no_cpu_fallback():
    from visualdet3d_b200.detectors import build_synthetic_stereo3d
    from visualdet3d_b200._lib import Vd3dError
    from visualdet3d_b200 import synth
    det, *_ = build_synthetic_stereo3d()
    l, r, P2, P3 = synth.synth_stereo_inputs(1, 32, 64)
    with pytest.raises(Vd3dError):
        det([l, r, P2, P3])


def test_product_does_not_import_oracle():
    import re
    bad = []
    for dp, _, fs in os.walk(os.path.join(ROOT, "visualdet3d_b200")):
        for f in fs:
            if f.endswith(".py"):
                txt = open(os.path.join(dp, f)).read()
                if re.search(r"^\s*(from|import)\s+(oracle|torch_port)", txt, flags=re.M):
                    bad.append(f)
    assert not bad, bad


def test_anchor_table_matches_oracle_bitwise():
    import numpy as np
    import torch_port as tp
    from visualdet3d_b200 import synth
    from visualdet3d_b200.anchors import AnchorTable
    pm, ps = synth.synth_priors(16, 3, ["Car", "Pedestrian"])
    cfg = synth.stereo3d_cfg("/x")
    for hw in [(96, 320), (288, 1280), (100, 330)]:
        a, ms, means = tp.build_anchors(hw, cfg["head"]["anchors_cfg"], pm, ps)
        t = AnchorTable(hw, cfg["head"]["anchors_cfg"], pm, ps, "cpu")
        assert torch.equal(t.anchors, a) and torch.equal(t.mean_std, ms) and torch.equal(t.means_z, means[:, :, 0])


@pytest.mark.parametrize("kind", ["Yolo3D", "GroundAwareYolo3D"])
def test_mono3d_registered_and_state_dict_keys_match_reference(kind):
    from visualdet3d_b200.plugin import DETECTOR_DICT
    from visualdet3d_b200.detectors import build_synthetic_mono3d
    assert kind in DETECTOR_DICT
    det, sd, cfg, _ = build_synthetic_mono3d(kind)
    ref = json.load(open(os.path.join(GOLDEN, f"{kind.lower()}_keys.json")))
    mine = {k: list(v.shape) for k, v in det.state_dict().items()}
    assert list(mine.keys()) == list(ref.keys()) and mine == ref
    with pytest.raises(NotImplementedError):
        det([torch.zeros(1, 3, 32, 32), None, torch.zeros(1, 3, 4)])          # 3-element list = training protocol


@pytest.mark.parametrize("kind", ["MonoFlex", "KM3D"])
def test_monoflex_registered_and_state_dict_keys_match_reference(kind):
    from visualdet3d_b200.plugin import DETECTOR_DICT
    from visualdet3d_b200.detectors import build_synthetic_monoflex
    assert "MonoFlex" in DETECTOR_DICT and "KM3D" in DETECTOR_DICT
    det, sd, cfg = build_synthetic_monoflex(name=kind)
    ref = json.load(open(os.path.join(GOLDEN, f"{kind.lower()}_keys.json")))
    mine = {k: list(v.shape) for k, v in det.state_dict().items()}
    assert list(mine.keys()) == list(ref.keys()) and mine == ref


def test_host_side_tile_and_layout_helpers():
    """Pure host entries of the C ABI (no GPU): the persistent conv engine's default tile width and the stem's padded row pitch."""
    from visualdet3d_b200 import _lib
    lib = _lib.load()
    for cout in (16, 24, 64, 72, 128, 144, 256, 288, 384, 608, 1152, 1408, 2048):
        bn = lib.vd3d_tc_pick_bn_persistent(cout)
        cp = (cout + 15) // 16 * 16
        assert bn % 16 == 0 and 16 <= bn <= 128
        n_tiles = (cp + bn - 1) // bn
        assert n_tiles == (cp + 127) // 128                      # as few tiles as 128 accumulator columns (the widest tile) allow ...
        assert n_tiles * bn - cp < 16 * n_tiles                  # ... split evenly (less than one 16-column granule of padding per tile)
    assert lib.vd3d_tc_pick_bn_persistent(1408) == 128 and lib.vd3d_tc_pick_bn_persistent(608) == 128 and lib.vd3d_tc_pick_bn_persistent(144) == 80
    assert lib.vd3d_tc_pick_bn_persistent(64) == 64
    # stem rows: `pad` zero pixels on the left, the image, and the 16-pixel window of the last output column; even pixel count
    for (W, KW, s, pad) in ((1280, 7, 2, 3), (320, 7, 2, 3), (53, 7, 2, 3), (96, 3, 2, 1)):
        Wp = lib.vd3d_stem_row_pitch(W, KW, s, pad)
        Wo = (W + 2 * pad - KW) // s + 1
        assert Wp % 2 == 0 and Wp >= W + pad and Wp >= s * (Wo - 1) + 16
    # the null-pointer / bad-argument paths return an error code and a message instead of launching anything
    assert lib.vd3d_conv2d_tc16_stem(None, None, 1, 8, 8, 16, 7, 7, 2, 3, 32, None, None, 1.0, None, None, None, None, 64, 64, 0, 1, None) != 0
    assert b"null pointer" in lib.vd3d_last_error()


def test_row_strip_host_helpers():
    """Pure host entries of the row-strip kernels (no GPU): padded row pitches of the fp16 row planes, and the argument checks that run before any launch."""
    from visualdet3d_b200 import _lib
    lib = _lib.load()
    # stem + pool: 5 leading zero pixels; 63 pooled columns (126 conv columns, 252 pixels, 2016 bytes) per strip, the last strip stages 264 pixels
    assert lib.vd3d_stem_pool_xoff() == 5
    for W in (30, 96, 320, 515, 1010, 1280):
        Wo = (W + 6 - 7) // 2 + 1
        Wq = (Wo - 1) // 2 + 1
        nstrips = (Wq + 62) // 63
        Wp = lib.vd3d_stem_pool_row_pitch(W)
        assert Wp % 2 == 0 and Wp >= W + 5 and Wp >= 252 * (nstrips - 1) + 264
    assert lib.vd3d_stem_pool_row_pitch(1280) == 252 * 5 + 264
    # row convs: 128 operand rows of 16 bytes per strip = 2048 bytes of input columns, + the filter row of the last operand row
    for (W, pc, KW, S, P, xoff) in ((1280, 8, 7, 1, 3, 4), (1280, 16, 3, 1, 1, 2), (1280, 16, 3, 2, 1, 2), (141, 16, 3, 2, 1, 2), (150, 8, 7, 1, 3, 4)):
        Wp = lib.vd3d_row_conv_pitch(W, pc, KW, S, P, xoff)
        pxb, Wo = pc * 2, (W + 2 * P - KW) // S + 1
        RS = S * pxb // 16
        nstrips = (Wo + 128 // RS - 1) // (128 // RS)
        KS = 2 if KW * pxb <= 64 else 4
        assert Wp % 4 == 0 and Wp >= W + xoff and Wp * pxb >= (xoff - P) * pxb + 2048 * (nstrips - 1) + 127 * 16 + KS * 32
    assert lib.vd3d_row_conv_pitch(1280, 12, 3, 1, 1, 2) < 0          # 24-byte pixels: not a whole number of 16-byte operand rows
    assert lib.vd3d_row_conv_pitch(1280, 16, 3, 1, 1, 0) < 0          # fewer leading zero pixels than the padding
    assert lib.vd3d_row_conv_pitch(1280, 16, 5, 1, 2, 2) < 0          # filter row wider than one 128-byte weight row
    assert lib.vd3d_row_conv(None, None, 1, 8, 8, 16, 2, 16, 3, 3, 1, 1, None, None, 1.0, None, 1, 16, None, None, None, 8, 0, 16, 0, None) != 0
    assert b"null pointer" in lib.vd3d_last_error()
    assert lib.vd3d_stem_pool_fused(None, None, 1, 8, 8, 16, None, None, 1.0, None, None, None, None, 64, 0, None) != 0
    assert b"null pointer" in lib.vd3d_last_error()
