"""CPU-side checks of the native MonoFlex head loss (visualdet3d_b200/monoflex_loss.py): the configuration from the shipped loss settings
and from a head, every refusal, the fixture's head outputs rebuilt from their seeds, the opt-in installer into the reference, and -- with
the reference present -- a rerun of the unmodified reference loss that reproduces tests/golden/monoflex_loss.npz bit for bit."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_fixture
from visualdet3d_b200 import monoflex_loss
from visualdet3d_b200.detectors import monoflex_cfg
from visualdet3d_b200.monoflex_loss import LossConfig

FX = load_fixture("monoflex_loss")
CASES = ["a", "b", "c"]


def golden_module():
    spec = importlib.util.spec_from_file_location("make_golden_monoflex_loss", os.path.join(GOLDEN, "make_golden_monoflex_loss.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


GEN = golden_module()


def case_inputs(fx, device):
    """(output, annotations, P2) of a fixture case on `device`; annotations with ind int64 and reg_mask bool as head_loss leaves them."""
    out = {k: v.to(device) for k, v in GEN.head_outputs(fx).items()}
    ann = {k: v.to(device) for k, v in GEN.annotations(fx).items()}
    ann["reg_mask"] = ann["reg_mask"].bool()
    return out, ann, torch.from_numpy(fx["P2"]).to(device)


def test_config_from_shipped_loss_cfg_and_head():
    c = LossConfig.from_loss_cfg(monoflex_cfg().head.loss_cfg)            # Monoflex_example: gamma, output_w only -> build_loss defaults
    assert c == LossConfig() and c.uncertainty_range == (-10.0, 10.0) and c.uncertainty_weight == 1.0
    c = LossConfig.from_loss_cfg(dict(uncertainty_range=[-3, 5], uncertainty_weight=0.5))
    assert c.uncertainty_range == (-3.0, 5.0) and c.uncertainty_weight == 0.5

    class Head:
        uncertainty_range = [-2, 2]
        uncertainty_weight = 2.0
    assert LossConfig.from_head(Head()) == LossConfig((-2.0, 2.0), 2.0)


def test_refusals():
    with pytest.raises(ValueError, match="uncertainty_range"):
        LossConfig.from_loss_cfg(dict(uncertainty_range=[1, -1]))
    out, ann, P2 = case_inputs(FX["b"], "cpu")
    with pytest.raises(RuntimeError, match="CUDA"):                       # no CPU path
        monoflex_loss.monoflex_head_loss(out, ann, P2)
    if not torch.cuda.is_available():
        return
    out, ann, P2 = case_inputs(FX["b"], "cuda")

    def refused(exc, match, out=out, ann=ann, P2=P2):
        with pytest.raises(exc, match=match):
            monoflex_loss.monoflex_head_loss(out, ann, P2)
    refused(RuntimeError, "float32", out=dict(out, dim=out["dim"].double()))
    refused(RuntimeError, "int64", ann=dict(ann, ind=ann["ind"].int()))
    refused(RuntimeError, "float32", ann=dict(ann, kp_detph_mask=ann["kp_detph_mask"].bool()))
    refused(ValueError, "channels", out=dict(out, hps=out["hps"][:, :18]))
    refused(ValueError, "does not match", out=dict(out, rot=out["rot"][:, :, :-1]))
    refused(ValueError, "does not match", out=dict(out, reg=out["reg"][:1]))
    refused(ValueError, "object rows", ann={**ann, **{k: torch.cat([v] * 9, 1) for k, v in ann.items() if k != "hm"}})
    refused(ValueError, "dep", ann=dict(ann, dep=ann["dep"][:, :-1]))
    refused(ValueError, "kp_detph_mask", ann=dict(ann, kp_detph_mask=ann["kp_detph_mask"][:, :, :2]))
    refused(ValueError, "P2", P2=P2[:, :, :3])


@pytest.mark.parametrize("case", CASES)
def test_fixture_inputs_rebuild(case):
    """The head outputs regenerate from the stored seed and edits, so the GPU tests feed the reference's inputs."""
    fx = FX[case]
    assert GEN.maps_sha(GEN.head_outputs(fx)) == str(fx["maps_sha"])
    hm = GEN.hm_target(fx)
    assert (hm == 1).any() == (case != "c")


def _reference():
    import refload
    if not refload.available():
        pytest.skip("reference package not available")
    return refload


def test_install_monoflex_loss_into_reference():
    _reference().load_reference()
    from visualDet3D.networks.heads import km3d_head, monoflex_head
    from visualDet3D.networks.heads import detection_3d_head
    from visualdet3d_b200 import plugin
    orig, km3d, anchor = monoflex_head.MonoFlexHead.loss, km3d_head.KM3DHead.loss, detection_3d_head.AnchorBasedDetection3DHead.loss
    try:
        fn = plugin.install_monoflex_loss_into_reference()
        assert fn is monoflex_loss.head_loss and monoflex_head.MonoFlexHead.loss is monoflex_loss.head_loss
        assert km3d_head.KM3DHead.loss is km3d                                # KM3D keeps its own loss
        assert detection_3d_head.AnchorBasedDetection3DHead.loss is anchor
    finally:
        monoflex_head.MonoFlexHead.loss = orig


@pytest.mark.parametrize("case", CASES)
def test_reference_rerun_matches_fixture(case):
    _reference().load_reference()
    from visualDet3D.networks.heads import monoflex_head
    assert monoflex_head.MonoFlexHead.loss.__module__ == monoflex_head.__name__      # the reference's own loss
    fx = dict(FX[case])
    ref = GEN.run_case(case, dict(GEN.CASES[case]))
    for k, v in fx.items():
        assert np.array_equal(np.asarray(ref[k]), v), k
