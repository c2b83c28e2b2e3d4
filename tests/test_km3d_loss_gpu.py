"""The native KM3D head loss on the GPU (csrc/km3d_loss.cu through visualdet3d_b200/km3d_loss.py) against the unmodified reference loss
(tests/golden/make_golden_km3d_loss.py): terms and totals within 1e-5 relative, gradients within 1e-5 of each map's max |.| and zero
wherever the reference's are -- coor_loss and the hps / dim gradients within 1e-5 plus twice the float32 reference's own measured distance
from a float64 restatement, which they are also checked against, and prob within 1e-4 (float64 overlap in the fixture) -- bit-identical
reruns and CUDA-graph replays, the fixed launch count, the backward of a single term, NaN losses for an index outside the map, and a
reference KM3DHead training step on the GPU with the reference's own compiled iou3d, with and without the native loss."""
import numpy as np
import pytest
import torch

from loss_harness import graph_replay_matches_eager, run_seam_worker
from test_km3d_loss_cpu import CASES, FX, GEN, case_inputs
from visualdet3d_b200 import _lib, km3d_loss
from visualdet3d_b200.km3d_loss import MAPS, TERMS, LossConfig

pytestmark = pytest.mark.gpu
LOSS_RTOL = 1e-5
GRAD_TOL = 1e-5       # of each gradient map's max |.|
# prob's gradient is sigmoid(prob) - box_score per row.  The fixture's box_score comes from a float64 BEV overlap (the host stand-in for the
# reference's overlap kernel); the device computes it in float32 like that kernel, on metre-scale corner coordinates.  The reference step
# (tests/workers/km3d_loss_step.py) checks it against the reference's own compiled kernel.
GRAD_TOL_MAP = {"prob": 1e-4}


def scatter_tol(fx, key):
    """coor_loss and the hps / dim gradients (which carry coor_loss's) through the least-squares solve: the fixture records how far the
    float32 reference itself lies from a float64 restatement (coor_ref_relerr, pos_ref_err_hps / _dim).  A float32 implementation as close
    to the exact value as the reference can differ from it by twice that, on top of the usual 1e-5."""
    base = LOSS_RTOL if key == "coor_loss" else GRAD_TOL
    err = float(fx["coor_ref_relerr"] if key == "coor_loss" else fx[f"pos_ref_err_{key}"])
    return base + 2.0 * err


def cfg(fx):
    return LossConfig(output_w=float(fx["W"]), rampup_length=float(GEN.RAMPUP))


def run(fx, epoch=GEN.GRAD_EPOCH):
    out, ann, P2 = case_inputs(fx, "cuda")
    for t in out.values():
        t.requires_grad_(True)
    loss, stats = km3d_loss.km3d_head_loss(out, ann, P2, epoch, cfg(fx))
    loss.backward()
    return loss, stats, {k: out[k].grad for k, _ in MAPS}


def close(got, ref, rtol=LOSS_RTOL):
    return abs(got - ref) <= rtol * abs(ref)


@pytest.mark.parametrize("case", CASES)
def test_terms_and_gradients_match_reference(case):
    fx = FX[case]
    loss, stats, grads = run(fx)
    assert set(stats) == set(TERMS) | {"loss", "total_loss"} and stats["total_loss"] is loss and len(stats) == 13
    assert torch.equal(stats["loss"], stats["box_score"])
    for i, key in enumerate(TERMS):
        got, ref = stats[key], float(fx["terms"][i])
        assert got.shape == () and got.dtype == torch.float32 and got.is_cuda
        assert close(float(got.detach()), ref, scatter_tol(fx, key) if key == "coor_loss" else LOSS_RTOL), (key, float(got), ref)
    assert close(float(loss.detach()), float(fx["total"]), LOSS_RTOL + float(fx["coor_ref_relerr"]))
    for name, _ in MAPS:
        g = grads[name].reshape(-1).cpu().numpy()
        idx, ref, gmax = fx[f"grad_{name}_idx"], fx[f"grad_{name}"], float(fx[f"grad_{name}_max"])
        if gmax == 0:
            assert not g.any(), name
            continue
        tol = scatter_tol(fx, name) if name in ("hps", "dim") else GRAD_TOL_MAP.get(name, GRAD_TOL)
        assert np.abs(g[idx] - ref).max() <= tol * gmax, (name, np.abs(g[idx] - ref).max(), gmax)
        assert abs(float(np.abs(g).max()) - gmax) <= tol * gmax, name
        if name not in ("hm", "hm_hp"):                           # zero wherever the reference's is
            others = np.ones(g.size, dtype=bool)
            others[idx] = False
            assert not g[others].any(), name


@pytest.mark.parametrize("case", CASES)
def test_position_loss_against_float64(case):
    """coor_loss and its hps / dim gradients against the float64 restatement: no further from the exact value than the float32 reference
    is (plus 1e-5)."""
    fx = FX[case]
    out, ann, P2 = case_inputs(fx, "cuda")
    for t in out.values():
        t.requires_grad_(True)
    _, stats = km3d_loss.km3d_head_loss(out, ann, P2, GEN.GRAD_EPOCH, cfg(fx))
    c64 = float(fx["coor64"])
    assert abs(float(stats["coor_loss"].detach()) - c64) <= (LOSS_RTOL + float(fx["coor_ref_relerr"])) * abs(c64)
    stats["coor_loss"].backward()
    for m in ("hps", "dim"):
        g = out[m].grad.reshape(-1).double().cpu().numpy()
        ref = np.zeros_like(g)
        ref[fx[f"pos64_{m}_idx"]] = fx[f"pos64_{m}"]
        err = np.abs(g - ref).max() / float(fx[f"grad_{m}_max"]) if float(fx[f"grad_{m}_max"]) > 0 else float(np.abs(g).max())
        assert err <= GRAD_TOL + float(fx[f"pos_ref_err_{m}"]), (m, err, float(fx[f"pos_ref_err_{m}"]))


@pytest.mark.parametrize("case", CASES)
def test_totals_across_the_rampup(case):
    fx = FX[case]
    out, ann, P2 = case_inputs(fx, "cuda")
    for e, ref in zip(GEN.EPOCHS, fx["totals"]):
        loss, _ = km3d_loss.km3d_head_loss(out, ann, P2, e, cfg(fx))
        assert close(float(loss), float(ref), LOSS_RTOL + float(fx["coor_ref_relerr"])), (e, float(loss), float(ref))


def test_two_runs_bit_identical():
    a = run(FX["a"])
    b = run(FX["a"])
    assert torch.equal(a[0], b[0])
    for k in TERMS:
        assert torch.equal(a[1][k], b[1][k])
    for k, _ in MAPS:
        assert torch.equal(a[2][k], b[2][k])


def test_launch_count_fixed():
    for case in CASES:
        out, ann, P2 = case_inputs(FX[case], "cuda")
        out["hm"].requires_grad_(True)
        _lib.launch_count_reset()
        loss, _ = km3d_loss.km3d_head_loss(out, ann, P2, 0, cfg(FX[case]))
        n_fwd = _lib.launch_count()
        loss.backward()
        assert n_fwd == 3 and _lib.launch_count() == 4            # hm, rows, combine; backward: one kernel


def test_cuda_graph_replay_bit_identical():
    fx = FX["b"]
    out, ann, P2 = case_inputs(fx, "cuda")
    for t in out.values():
        t.requires_grad_(True)

    def step():
        for t in out.values():
            t.grad = None
        loss, stats = km3d_loss.km3d_head_loss(out, ann, P2, GEN.GRAD_EPOCH, cfg(fx))
        loss.backward()
        return [loss] + [stats[k] for k in TERMS] + [out[k].grad for k, _ in MAPS]

    graph_replay_matches_eager(step)


def test_backward_of_a_single_term():
    """d coor_loss alone touches only hps and dim; d hm_hp_loss alone only hm_hp, the same gradient the total gives it."""
    fx = FX["a"]
    _, _, grads = run(fx)
    out, ann, P2 = case_inputs(fx, "cuda")
    for t in out.values():
        t.requires_grad_(True)
    _, stats = km3d_loss.km3d_head_loss(out, ann, P2, GEN.GRAD_EPOCH, cfg(fx))
    stats["coor_loss"].backward(retain_graph=True)
    assert out["hps"].grad.any() and out["dim"].grad.any()
    for k, _ in MAPS:
        if k not in ("hps", "dim"):
            assert not out[k].grad.any(), k
    for t in out.values():
        t.grad = None
    stats["hm_hp_loss"].backward()
    assert torch.equal(out["hm_hp"].grad, grads["hm_hp"])
    for k, _ in MAPS:
        if k != "hm_hp":
            assert not out[k].grad.any(), k


@pytest.mark.parametrize("key", ["ind", "hp_ind"])
def test_index_outside_the_map_gives_nan(key):
    fx = FX["b"]
    out, ann, P2 = case_inputs(fx, "cuda")
    H, W = int(fx["H"]), int(fx["W"])
    ann[key] = ann[key].clone()
    ann[key][1, 3] = H * W
    loss, stats = km3d_loss.km3d_head_loss(out, ann, P2, 0, cfg(fx))
    assert torch.isnan(loss).item() and all(torch.isnan(stats[k]).item() for k in TERMS)


def test_reference_head_training_step():
    out = run_seam_worker("km3d_loss_step.py")
    assert out["native_bound"] and out["reference_iou3d_kernel"] and out["same_params"] and out["n_grads"] >= 36
    # within 1e-5, plus twice the reference's own scatter between two draws of its solve jitter
    for k, v in out["loss_rel"].items():
        assert v <= LOSS_RTOL + 2.0 * out["ref_scatter_loss"][k], (k, v, out["ref_scatter_loss"][k])
    for k, v in out["grad_err"].items():
        assert v <= GRAD_TOL + 2.0 * out["ref_scatter_grad"][k], (k, v, out["ref_scatter_grad"][k])
