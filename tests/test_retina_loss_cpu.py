"""CPU-side checks of the native RetinaNet head loss (visualdet3d_b200/retina_loss.py): configuration parsing from the shipped config and
from a reference head, every refusal, the opt-in installer into the reference, the project's anchor table against the reference's
`Anchors`, and -- with the reference present -- a rerun of the unmodified reference loss that reproduces tests/golden/retina_loss.npz bit
for bit."""
import hashlib
import importlib.util
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_fixture
from visualdet3d_b200 import retina_loss, synth
from visualdet3d_b200.anchors import grid_anchors
from visualdet3d_b200.retina_loss import LossConfig

FX = load_fixture("retina_loss")
CASES = ["train", "edge", "argmax", "nopos"]


def anchor_table(H, W):
    a = synth.retinanet_cfg().head.anchors_cfg
    return torch.from_numpy(grid_anchors((H, W), a["pyramid_levels"], a["strides"], a["sizes"], a["ratios"], a["scales"]).astype(np.float32))


def case_config(fx) -> LossConfig:
    return LossConfig.from_loss_cfg(json.loads(str(fx["loss_cfg"])), int(fx["C"]), fx["target_means"].tolist(), fx["target_stds"].tolist())


def case_inputs(fx, device):
    """(cls_scores, reg_preds, anchors [1, N, 4], annotations, LossConfig) of a fixture case on `device`."""
    B, H, W, C = int(fx["B"]), int(fx["H"]), int(fx["W"]), int(fx["C"])
    anchors = anchor_table(H, W)
    cls, reg = synth.retina_head_outputs(B, anchors.shape[0], C, seed=int(fx["seed"]))
    return cls.to(device), reg.to(device), anchors[None].to(device), torch.from_numpy(fx["ann"]).to(device), case_config(fx)


def _sha(t):
    return hashlib.sha256(np.ascontiguousarray(t.detach().cpu().numpy().astype(np.float32)).tobytes()).hexdigest()


def test_config_from_shipped_loss_cfg():
    hc = synth.retinanet_cfg().head
    c = LossConfig.from_loss_cfg(hc.loss_cfg, hc.num_classes, hc.target_means, hc.target_stds)
    assert (c.fg_iou_threshold, c.bg_iou_threshold, c.min_iou_threshold) == (0.5, 0.4, 0.0)
    assert c.match_low_quality and c.gt_max_assign_all and c.gamma == 2.0 and c.balance_weights == (1.0,)
    p = c.params()
    assert p.dtype == np.float32 and p.shape == (12 + 3,)
    assert np.array_equal(p, np.float32([0.5, 0.4, 0.0, 2.0, 0.0, 0.0, 0.0, 0.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0]))
    # build_loss's default balance_weights=0 is a 0-d tensor: one weight, broadcast over the classes
    d = LossConfig.from_loss_cfg({}, 2)
    assert (d.bg_iou_threshold, d.gamma, d.balance_weights, d.target_stds) == (0.0, 0.0, (0.0,), (1.0, 1.0, 1.0, 1.0))
    assert d.params()[12:].tolist() == [0.0, 0.0]
    e = case_config(FX["edge"])
    assert e.balance_weights == (0.5, 2.0, 4.0) and e.gamma == 0.0 and e.params()[8:12].tolist() == np.float32([0.2, 0.25, 0.5, 0.4]).tolist()
    assert not case_config(FX["argmax"]).gt_max_assign_all and not case_config(FX["nopos"]).match_low_quality


def test_refusals():
    with pytest.raises(ValueError, match="balance_weights"):
        LossConfig.from_loss_cfg(dict(balance_weights=[1.0, 2.0]), 3)
    with pytest.raises(ValueError, match="num_classes"):
        LossConfig(num_classes=65)
    with pytest.raises(ValueError, match="target_means"):
        LossConfig.from_loss_cfg({}, 3, target_means=[0.0] * 3)
    cls, reg, anchors, ann, cfg = case_inputs(FX["edge"], "cpu")
    B, N, C = cls.shape
    bad = [(cls, reg[:, :, :3], anchors, ann, "reg_preds"),                         # reg_preds not [B, N, 4]
           (cls, reg, anchors[:, :-1], ann, "anchors"),                              # anchors that do not hold N boxes
           (cls, reg, anchors, ann[:, :, :4], "annotations"),                        # K < 5
           (cls, reg, anchors, torch.full((B, 513, 12), -1.0), "annotation rows"),   # more rows than the kernels hold
           (cls[:, :, :2], reg, anchors, ann, "columns")]                            # a class count other than the head's
    for c, r, a, m, what in bad:
        with pytest.raises(ValueError, match=what):
            retina_loss.retinanet_head_loss(c, r, a, m, cfg)
    with pytest.raises(RuntimeError, match="float32"):
        retina_loss.retinanet_head_loss(cls.double(), reg, anchors, ann, cfg)
    with pytest.raises(RuntimeError, match="CUDA"):                                 # no CPU path
        retina_loss.retinanet_head_loss(cls, reg, anchors, ann, cfg)
    with pytest.raises(RuntimeError, match="CUDA"):
        retina_loss.assignment(cls, reg, anchors, ann, cfg)


def _reference():
    import refload
    if not refload.available():
        pytest.skip("reference package not available")
    refload.load_reference()
    return refload


def _golden_module():
    spec = importlib.util.spec_from_file_location("make_golden_retina_loss", os.path.join(GOLDEN, "make_golden_retina_loss.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_config_from_reference_head():
    _reference()
    gm = _golden_module()
    head = gm.build_head(gm.CASES["edge"])
    c = LossConfig.from_head(head)
    assert c == case_config(FX["edge"])
    assert retina_loss._head_config(head) is retina_loss._head_config(head)          # cached on the head
    with torch.no_grad():
        head.loss_cls.balance_weights.mul_(2.0)                                      # an in-place write invalidates the cache
    assert retina_loss._head_config(head).balance_weights == (1.0, 4.0, 8.0)


def test_install_retinanet_loss_into_reference():
    _reference()
    from visualDet3D.networks.heads import retinanet_head as ref_head
    from visualDet3D.networks.utils import registry
    from visualdet3d_b200 import plugin
    orig = ref_head.RetinanetHead.loss
    det = registry.DETECTOR_DICT["RetinaNet"]
    try:
        fn = plugin.install_retinanet_loss_into_reference()
        assert fn is retina_loss.head_loss and ref_head.RetinanetHead.loss is retina_loss.head_loss
        assert registry.DETECTOR_DICT["RetinaNet"] is det                           # the detector registry is untouched
    finally:
        ref_head.RetinanetHead.loss = orig


@pytest.mark.parametrize("hw", [(288, 1280), (96, 320)])
def test_anchor_table_matches_reference(hw):
    _reference()
    from visualDet3D.networks.heads.anchors import Anchors
    a = synth.retinanet_cfg().head.anchors_cfg
    ref = Anchors(preprocessed_path=None, readConfigFile=False, **dict(a))(torch.zeros(1, 3, *hw))
    ours = anchor_table(*hw)
    assert ref.shape == (1, ours.shape[0], 4) and ref.dtype == torch.float32
    assert torch.equal(ref[0], ours)


@pytest.mark.parametrize("case", CASES)
def test_fixture_inputs_rebuild(case):
    fx = FX[case]
    cls, reg, anchors, ann, _ = case_inputs(fx, "cpu")
    assert _sha(anchors[0]) == str(fx["anchors_sha"])
    assert fx["assign"].shape == cls.shape[:2] and fx["counts"].sum(1).tolist() == [cls.shape[1]] * cls.shape[0]


@pytest.mark.parametrize("case", CASES)
def test_reference_rerun_matches_fixture(case):
    _reference()
    from visualDet3D.networks.heads import retinanet_head as ref_head
    assert ref_head.RetinanetHead.loss.__module__ == ref_head.__name__                 # the reference's own loss
    out = _golden_module().run_case(case)
    fx = FX[case]
    assert sorted(out) == sorted(fx)
    for k, v in out.items():
        v = np.asarray(v)
        assert v.dtype == fx[k].dtype and v.shape == fx[k].shape and v.tobytes() == fx[k].tobytes(), k
