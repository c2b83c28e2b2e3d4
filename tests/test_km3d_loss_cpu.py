"""CPU-side checks of the native KM3D head loss (visualdet3d_b200/km3d_loss.py): the configuration from the shipped loss settings and
from a head, exp_rampup, every refusal, the fixture's own consistency (head outputs rebuilt from their seeds, self-consistent targets),
the opt-in installer into the reference, and -- with the reference present -- a rerun of the unmodified reference loss that reproduces
tests/golden/km3d_loss.npz."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_fixture
from visualdet3d_b200 import km3d_loss
from visualdet3d_b200.detectors import km3d_cfg
from visualdet3d_b200.km3d_loss import LossConfig

FX = load_fixture("km3d_loss")
CASES = ["a", "b", "c", "d", "e"]


def golden_module():
    spec = importlib.util.spec_from_file_location("make_golden_km3d_loss", os.path.join(GOLDEN, "make_golden_km3d_loss.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


GEN = golden_module()


def case_inputs(fx, device):
    """(output, annotations, P2) of a fixture case on `device`."""
    out = {k: v.to(device) for k, v in GEN.head_outputs(fx).items()}
    ann = {k: v.to(device) for k, v in GEN.annotations(fx).items()}
    return out, ann, torch.from_numpy(fx["P2"]).to(device)


def test_config_from_shipped_loss_cfg_and_head():
    c = LossConfig.from_loss_cfg(km3d_cfg().head.loss_cfg)                  # KM3D_example: output_w 320, rampup_length 100
    assert c == LossConfig(output_w=320.0, rampup_length=100.0)
    assert LossConfig.from_loss_cfg({}) == LossConfig(1280.0, 100.0)         # build_loss defaults

    class PL:
        output_w = 80

    class Head:
        position_loss = PL()
        rampup_length = 7
    assert LossConfig.from_head(Head()) == LossConfig(80.0, 7.0)


def test_exp_rampup_matches_reference_formula():
    c = LossConfig(rampup_length=100)
    assert c.exp_rampup(0) == float(np.exp(-5.0))
    assert c.exp_rampup(37) == float(np.exp(-5.0 * 0.63 * 0.63))
    assert c.exp_rampup(100) == 1.0 and c.exp_rampup(250) == 1.0


def test_refusals():
    with pytest.raises(ValueError, match="output_w"):
        LossConfig(output_w=0)
    out, ann, P2 = case_inputs(FX["b"], "cpu")
    with pytest.raises(RuntimeError, match="CUDA"):                       # no CPU path
        km3d_loss.km3d_head_loss(out, ann, P2)
    if not torch.cuda.is_available():
        return
    out, ann, P2 = case_inputs(FX["b"], "cuda")

    def refused(exc, match, out=out, ann=ann, P2=P2):
        with pytest.raises(exc, match=match):
            km3d_loss.km3d_head_loss(out, ann, P2)
    refused(RuntimeError, "float32", out=dict(out, dim=out["dim"].double()))
    refused(RuntimeError, "int64", ann=dict(ann, hp_ind=ann["hp_ind"].int()))
    refused(ValueError, "channels", out=dict(out, hps=out["hps"][:, :16]))
    refused(ValueError, "does not match", out=dict(out, rot=out["rot"][:, :, :-1]))
    refused(ValueError, "hm_hp", ann=dict(ann, hm_hp=ann["hm_hp"][:, :8]))
    refused(ValueError, "object rows", ann={**ann, "ind": torch.cat([ann["ind"]] * 9, 1)})
    refused(ValueError, "hp_offset", ann=dict(ann, hp_offset=ann["hp_offset"][:, :-1]))
    refused(ValueError, "location", ann=dict(ann, location=ann["location"][:, :, :2]))
    refused(ValueError, "P2", P2=P2[:, :, :3])


@pytest.mark.parametrize("case", CASES)
def test_fixture_consistency(case):
    """The head outputs regenerate from the stored seed and edits, and the targets hang together: the keypoint targets are the boxes'
    projections relative to ind, hp_ind / hp_offset address the same keypoints, the peaks are 1 where the cases say so."""
    fx = FX[case]
    assert GEN.maps_sha(GEN.head_outputs(fx)) == str(fx["maps_sha"])
    B, C, H, W, K = (int(fx[k]) for k in ("B", "C", "H", "W", "K"))
    ann = GEN.annotations(fx)
    # each heatmap's num_pos is batch-wide: d has no exact 1 in hm only, e in hm_hp only
    assert (ann["hm"] == 1).any() == (case not in ("c", "d")) and (ann["hm_hp"] == 1).any() == (case not in ("c", "e"))
    for b in range(B):
        for k in range(K):
            if not fx["reg_mask"][b, k]:
                continue
            loc = fx["location"][b, k].astype(np.float64)
            assert loc[2] > 1.0                                              # in front of the camera
            kp = GEN.project(fx["P2"][b].astype(np.float64), GEN.corners(*loc, *fx["dim"][b, k], float(fx["ori"][b, k, 0]))) / 4
            cy, cx = divmod(int(fx["ind"][b, k]), W)
            if not (case == "b" and b == 1 and k == 1):                     # the disjoint row's location was moved on purpose
                assert np.allclose(fx["hps"][b, k].reshape(9, 2), kp - [cx, cy], atol=1e-3)
            for j in range(9):
                r = k * 9 + j
                if fx["hp_mask"][b, r]:
                    vy, vx = divmod(int(fx["hp_ind"][b, r]), W)
                    assert np.allclose(fx["hp_offset"][b, r], fx["hps"][b, k].reshape(9, 2)[j] + [cx, cy] - [vx, vy], atol=1e-3)
    assert fx["totals"][0] <= fx["totals"][1] <= fx["totals"][2]


def test_annotations_not_mutated():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    out, ann, P2 = case_inputs(FX["a"], "cuda")
    before = {k: v.clone() for k, v in ann.items()}
    km3d_loss.km3d_head_loss(out, ann, P2, 37, LossConfig(output_w=float(FX["a"]["W"])))
    torch.cuda.synchronize()
    for k, v in ann.items():
        assert torch.equal(v, before[k]), k


def _reference():
    import refload
    if not refload.available():
        pytest.skip("reference package not available")
    return refload


def test_install_km3d_loss_into_reference():
    _reference().load_reference()
    from visualDet3D.networks.heads import km3d_head, monoflex_head
    from visualDet3D.networks.heads import detection_3d_head
    from visualdet3d_b200 import plugin
    orig, mono, anchor = km3d_head.KM3DHead.loss, monoflex_head.MonoFlexHead.loss, detection_3d_head.AnchorBasedDetection3DHead.loss
    try:
        fn = plugin.install_km3d_loss_into_reference()
        assert fn is km3d_loss.head_loss and km3d_head.KM3DHead.loss is km3d_loss.head_loss
        assert monoflex_head.MonoFlexHead.loss is mono and mono is not km3d_loss.head_loss   # MonoFlex keeps its own loss
        assert detection_3d_head.AnchorBasedDetection3DHead.loss is anchor
    finally:
        km3d_head.KM3DHead.loss = orig


@pytest.mark.parametrize("case", CASES)
def test_reference_rerun_matches_fixture(case):
    _reference().load_reference()
    from visualDet3D.networks.heads import km3d_head
    assert km3d_head.KM3DHead.loss.__module__ == km3d_head.__name__      # the reference's own loss
    fx = dict(FX[case])
    ref = GEN.run_case(case, dict(GEN.CASES[case]))
    for k, v in fx.items():
        r = np.asarray(ref[k])
        if k == "maps_sha" or not np.issubdtype(v.dtype, np.floating):
            assert np.array_equal(r, v), k
        else:                                                             # float32 rounding of the host's threaded reductions
            assert r.shape == v.shape and np.allclose(r, v, rtol=1e-5, atol=1e-6 * max(1.0, float(np.abs(v).max(initial=0)))), k
