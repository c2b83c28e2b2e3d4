"""CPU-side checks of the native 3-D anchor head loss (visualdet3d_b200/anchor_loss.py): configuration parsing and every refusal, the
opt-in installer into the reference, the fixture's inputs rebuilt by the project's own anchor table, and -- with the reference present --
a rerun of the unmodified reference loss that reproduces tests/golden/anchor_loss.npz bit for bit."""
import hashlib
import importlib.util
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_fixture
from visualdet3d_b200 import anchor_loss, synth
from visualdet3d_b200.anchor_loss import LossConfig
from visualdet3d_b200.anchors import AnchorTable

FX = load_fixture("anchor_loss")
CASES = ["a", "b", "c"]


def head_cfg(kind: str):
    """The head config of a fixture case (tests/golden/make_golden_anchor_loss.py::head_setup)."""
    return synth.mono3d_cfg("", "GroundAwareYolo3D").head if kind == "Yolo3D" else synth.stereo3d_cfg("").head


def case_inputs(fx, device):
    """(cls_scores, reg_preds, anchors dict, annotations, loss_cfg) of a fixture case on `device`."""
    hc = head_cfg(str(fx["kind"]))
    B, H, W = int(fx["B"]), int(fx["H"]), int(fx["W"])
    table = AnchorTable((H, W), hc.anchors_cfg, fx["pm"], fx["ps"], device)
    mask = np.unpackbits(fx["mask_bits"])[:B * table.N].reshape(B, table.N).astype(bool)
    cls, reg = synth.synth_head_outputs(B, table.N, hc.num_classes, seed=int(fx["seed"]))
    anchors = dict(anchors=table.anchors[None], mask=torch.from_numpy(mask).to(device), anchor_mean_std_3d=table.mean_std)
    return cls.to(device), reg.to(device), anchors, torch.from_numpy(fx["ann"]).to(device), hc.loss_cfg


def _sha(t):
    return hashlib.sha256(np.ascontiguousarray(t.detach().cpu().numpy().astype(np.float32)).tobytes()).hexdigest()


def test_config_from_shipped_loss_cfgs():
    c = LossConfig.from_loss_cfg(synth.stereo3d_cfg("").head.loss_cfg, 2)
    assert (c.fg_iou_threshold, c.bg_iou_threshold, c.min_iou_threshold) == (0.5, 0.4, 0.0)
    assert c.match_low_quality and c.gt_max_assign_all and c.focal_loss_gamma == 2.0 and c.l1_regression_alpha == 25.0
    assert c.balance_weights == (20.0, 40.0) and c.regression_weight[6] == 12.0 and len(c.regression_weight) == 13
    p = c.params()
    assert p.dtype == np.float32 and p.shape == (7 + 2 + 13,)
    assert p[4] == np.float32(1 / 25) and p[5] == np.float32(12.5) and p[6] == np.float32(0.02)
    y = LossConfig.from_loss_cfg(synth.mono3d_cfg("", "GroundAwareYolo3D").head.loss_cfg, 1)
    assert not y.match_low_quality and y.balance_weights == (20.0,) and y.regression_weight[6] == 3.0
    # one balance weight is broadcast over the classes
    assert LossConfig(num_classes=3, balance_weights=(5.0,)).params()[7:10].tolist() == [5.0, 5.0, 5.0]
    # the reference's _assign / build_loss defaults
    d = LossConfig.from_loss_cfg({}, 1)
    assert (d.bg_iou_threshold, d.focal_loss_gamma, d.l1_regression_alpha, d.balance_weights) == (0.0, 0.0, 9.0, (0.0,))


def test_refusals():
    lc = dict(synth.stereo3d_cfg("").head.loss_cfg)
    with pytest.raises(ValueError, match="decode_before_loss"):
        LossConfig.from_loss_cfg(dict(lc, decode_before_loss=True), 2)
    with pytest.raises(ValueError, match="balance_weight"):
        LossConfig.from_loss_cfg(dict(lc, balance_weight=[1.0, 2.0, 3.0]), 2)
    with pytest.raises(ValueError, match="regression_weight"):
        LossConfig.from_loss_cfg(dict(lc, regression_weight=[1.0] * 12), 2)
    with pytest.raises(ValueError, match="num_classes"):
        LossConfig(num_classes=9, balance_weights=(1.0,))
    cls, reg, anchors, ann, loss_cfg = case_inputs(FX["c"], "cpu")
    with pytest.raises(RuntimeError, match="CUDA"):                       # no CPU path
        anchor_loss.anchor3d_head_loss(cls, reg, anchors, ann, loss_cfg)
    with pytest.raises(RuntimeError, match="CUDA"):
        anchor_loss.assignment(cls, reg, anchors, ann, loss_cfg)


@pytest.mark.parametrize("case", CASES)
def test_fixture_inputs_rebuild(case):
    """The project's anchor table gives the reference's anchors and priors bit for bit, so the GPU tests feed the same inputs."""
    fx = FX[case]
    cls, reg, anchors, ann, _ = case_inputs(fx, "cpu")
    assert _sha(anchors["anchors"][0]) == str(fx["anchors_sha"])
    assert _sha(anchors["anchor_mean_std_3d"]) == str(fx["mean_std_sha"])
    assert fx["assign"].shape == tuple(anchors["mask"].shape)
    assert ((fx["assign"] == -2) == ~anchors["mask"].numpy()).all()


def _reference():
    import refload
    if not refload.available():
        pytest.skip("reference package not available")
    return refload


def test_install_loss_into_reference():
    _reference().load_reference()
    from visualDet3D.networks.detectors.yolomono3d_detector import GroundAwareHead
    from visualDet3D.networks.heads import detection_3d_head as ref_head
    from visualdet3d_b200 import plugin
    orig = ref_head.AnchorBasedDetection3DHead.loss
    try:
        fn = plugin.install_loss_into_reference()
        assert fn is anchor_loss.head_loss
        assert ref_head.StereoHead.loss is anchor_loss.head_loss
        assert GroundAwareHead.loss is anchor_loss.head_loss
    finally:
        ref_head.AnchorBasedDetection3DHead.loss = orig


def _golden_module():
    spec = importlib.util.spec_from_file_location("make_golden_anchor_loss", os.path.join(GOLDEN, "make_golden_anchor_loss.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("case", CASES)
def test_reference_rerun_matches_fixture(case, tmp_path):
    _reference().load_reference()
    from visualDet3D.networks.heads import detection_3d_head as ref_head
    assert ref_head.AnchorBasedDetection3DHead.loss.__module__ == ref_head.__name__      # the reference's own loss
    fx = FX[case]
    head, *_ = _golden_module().build_head(str(fx["kind"]), str(tmp_path))
    cls, reg, anchors, ann, _ = case_inputs(fx, "cpu")
    ref_anchors = head.get_anchor(torch.zeros(int(fx["B"]), 3, int(fx["H"]), int(fx["W"])), torch.from_numpy(fx["P2"]))
    assert torch.equal(ref_anchors["mask"], anchors["mask"])
    cls.requires_grad_(True)
    reg.requires_grad_(True)
    c, r, d = head.loss(cls, reg, ref_anchors, ann, torch.from_numpy(fx["P2"]))
    (c + r).sum().backward()
    assert c.detach().numpy().tobytes() == fx["cls_loss"].tobytes()
    assert r.detach().numpy().tobytes() == fx["reg_loss"].tobytes()
    assert d["total_loss"].detach().numpy().tobytes() == fx["total_loss"].tobytes()
    C1 = cls.shape[-1]
    assert np.array_equal(reg.grad.reshape(-1, 12).numpy()[fx["grad_reg_rows"]], fx["grad_reg"])
    assert np.array_equal(cls.grad.reshape(-1, C1).numpy()[fx["grad_cls_rows"]], fx["grad_cls"])
