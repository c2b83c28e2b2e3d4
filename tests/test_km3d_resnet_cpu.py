"""KM3D / MonoFlex on the ResNet CenterNet core, without a GPU: the parameter layout against the reference's, the backbone rules of
KM3DCoreP, the exactness of the sub-pixel phase packing of the transposed conv, and the oracle's ResNet core against the reference
fixtures (tests/golden/make_golden_km3d_resnet.py)."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN, load_fixture, subsample_like
import centernet_resnet_oracle as ro


def _shapes(det):
    return {k: list(v.shape) for k, v in det.state_dict().items()}


@pytest.mark.parametrize("kind,keys", [("KM3D", "km3d_resnet_keys.json"), ("MonoFlex", "monoflex_resnet_keys.json")])
def test_state_dict_keys_and_shapes_equal_the_reference(kind, keys):
    from visualdet3d_b200.detectors.centernet import km3d_example_cfg, monoflex_resnet_cfg
    from visualdet3d_b200.plugin import DETECTOR_DICT
    det = DETECTOR_DICT[kind](km3d_example_cfg() if kind == "KM3D" else monoflex_resnet_cfg())
    ref = json.load(open(os.path.join(GOLDEN, keys)))
    assert _shapes(det) == ref


def test_backbone_rules():
    from visualdet3d_b200.detectors import modules as M
    from visualdet3d_b200.detectors.centernet import KM3DCoreP, km3d_example_cfg
    from visualdet3d_b200.plugin import DETECTOR_DICT
    cfg = km3d_example_cfg()
    assert "name" not in cfg.backbone
    det = DETECTOR_DICT["KM3D"](cfg)                         # KM3D_example as shipped (pretrained=False): a ResNet-18 core
    assert isinstance(det.core.backbone, M.ResNetP) and det.core.backbone.depth == 18 and det.core.backbone_name == "resnet"
    assert [type(m).__name__ for m in det.core.deconv_layers] == ["ConvTranspose2d", "BatchNorm2d", "ReLU"] * 3
    for i in (0, 3, 6):
        w = det.core.deconv_layers[i].weight
        assert float(w.detach().std()) < 0.002                          # the reference's normal_(std=0.001) init
    assert isinstance(KM3DCoreP(dict(cfg.backbone, depth=34)).backbone, M.ResNetP)
    with pytest.raises(ValueError, match="2024"):
        KM3DCoreP(dict(cfg.backbone, depth=50))
    with pytest.raises(ValueError, match="stage 3"):
        KM3DCoreP(dict(cfg.backbone, out_indices=(1, 2)))
    with pytest.raises(NotImplementedError):
        KM3DCoreP(dict(cfg.backbone, name="vit"))
    from visualdet3d_b200.detectors.centernet import km3d_cfg
    assert DETECTOR_DICT["KM3D"](km3d_cfg()).core.backbone_name == "dla"


def test_transposed_conv_refused_off_the_fp16_split_engine(monkeypatch):
    from visualdet3d_b200 import engine as E
    from visualdet3d_b200._lib import Vd3dError
    monkeypatch.setenv("VD3D_CONV_ENGINE", "tc")
    with pytest.raises(Vd3dError, match="fp16-split"):
        E.ConvTransposeLayer(torch.randn(64, 32, 4, 4), device="cpu")


def _phases_from_matrix(m, Cin, Cout, x):
    """Run the packed [4 Cout][4 cin_pad] matrix as four 2x2 convs on x (float64) and interleave them."""
    B, _, H, W = x.shape
    cin_pad = m.shape[1] // 4
    y = torch.zeros(B, Cout, 2 * H, 2 * W, dtype=torch.float64)
    for r in (0, 1):
        for s in (0, 1):
            wl = m[(2 * r + s) * Cout:(2 * r + s + 1) * Cout].view(Cout, 2, 2, cin_pad)[..., :Cin].permute(0, 3, 1, 2)
            assert float(m[(2 * r + s) * Cout:(2 * r + s + 1) * Cout].view(Cout, 4, cin_pad)[..., Cin:].abs().sum()) == 0.0
            xp = F.pad(x, (1 - s, s, 1 - r, r))               # tap origin (1 - r, 1 - s); the far edge reads zeros
            y[:, :, r::2, s::2] = F.conv2d(xp, wl)
    return y


@pytest.mark.parametrize("H,W", [(1, 1), (1, 6), (5, 1), (3, 5), (7, 13), (4, 8)])
def test_phase_packing_is_exact(H, W):
    """On the CPU in float64: the four packed 2x2 phase convs, interleaved, equal F.conv_transpose2d(4, stride 2, padding 1) followed by
    the eval-mode BatchNorm, to rounding; odd sizes and H = 1 / W = 1 included."""
    from visualdet3d_b200 import engine as E
    g = torch.Generator().manual_seed(H * 100 + W)
    Cin, Cout, B = 20, 24, 2
    wt = torch.randn(Cin, Cout, 4, 4, generator=g, dtype=torch.float64)
    bn = dict(weight=torch.rand(Cout, generator=g, dtype=torch.float64) + 0.5, bias=torch.randn(Cout, generator=g, dtype=torch.float64),
              running_mean=torch.randn(Cout, generator=g, dtype=torch.float64), running_var=torch.rand(Cout, generator=g, dtype=torch.float64) + 0.5)
    x = torch.randn(B, Cin, H, W, generator=g, dtype=torch.float64)
    ref = F.batch_norm(F.conv_transpose2d(x, wt, None, stride=2, padding=1), bn["running_mean"], bn["running_var"], bn["weight"], bn["bias"],
                       training=False, eps=1e-5)
    wf, bf = E.fold_bn_transposed(wt, None, bn)
    m = E.convtranspose_phase_matrix(wf, 64)
    assert tuple(m.shape) == (4 * Cout, 4 * 64)
    got = _phases_from_matrix(m, Cin, Cout, x) + bf.view(1, -1, 1, 1)
    assert float((got - ref).abs().max()) < 1e-12 * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize("tag", ["km3d_resnet_96x320", "km3d_resnet_192x640", "monoflex_resnet_96x320"])
def test_oracle_resnet_core_matches_reference(tag):
    """The oracle's ResNet CenterNet core (tests/centernet_resnet_oracle.py) with torch_port's decodes against the reference's fixtures (same bars as the DLA oracle tests)."""
    from visualdet3d_b200 import synth
    from visualdet3d_b200.detectors.centernet import km3d_example_cfg, monoflex_resnet_cfg
    km3d = tag.startswith("km3d")
    fx = load_fixture(tag)
    H, W, B, seed = [int(v) for v in fx["meta"]]
    shapes = json.load(open(os.path.join(GOLDEN, ("km3d" if km3d else "monoflex") + "_resnet_keys.json")))
    sd = synth.synth_state_dict(shapes, seed)
    cfg = km3d_example_cfg(score_thr=0.1) if km3d else monoflex_resnet_cfg()
    img, P2 = synth.synth_mono_inputs(B, H, W, seed=1)
    st = {}
    outs = (ro.km3d_forward if km3d else ro.monoflex_forward)(sd, img, P2, cfg, st)
    np.testing.assert_allclose(subsample_like(st["features"], fx["features"]), fx["features"]["samples"], atol=2e-4)
    for n in cfg["head"]["layer_cfg"]["head_dict"]:
        np.testing.assert_allclose(subsample_like(st["heads"][n], fx["head_" + n]), fx["head_" + n]["samples"], atol=5e-4, err_msg=n)
    for b in range(B):
        s, bx, ci, _ = outs[b]
        assert len(s) == len(fx[f"scores_{b}"]) and len(s) > 3
        np.testing.assert_array_equal(ci.numpy(), fx[f"cls_{b}"])
        np.testing.assert_allclose(s.numpy(), fx[f"scores_{b}"], atol=1e-4)
        # KM3D: the reference jitters A^T A by 1e-8 randn before inverting it (rtm3d_utils.py:447)
        np.testing.assert_allclose(bx.numpy(), fx[f"bboxes_{b}"], atol=2e-3 if km3d else 1e-3, rtol=1e-4 if km3d else 1e-5)
