"""The native MonoFlex head loss on the GPU (csrc/monoflex_loss.cu through visualdet3d_b200/monoflex_loss.py) against the unmodified
reference loss (tests/golden/make_golden_monoflex_loss.py): terms and total within 1e-5 relative, gradients within 1e-5 of each map's max
|.| and zero wherever the reference's are, bit-identical reruns and CUDA-graph replays, the fixed launch count, NaN losses for an ind
outside the map, and a reference MonoFlexHead training step with the native loss installed."""
import numpy as np
import pytest
import torch

from loss_harness import graph_replay_matches_eager, run_seam_worker
from test_monoflex_loss_cpu import CASES, FX, case_inputs
from visualdet3d_b200 import _lib, monoflex_loss
from visualdet3d_b200.monoflex_loss import MAPS, TERMS

pytestmark = pytest.mark.gpu
LOSS_RTOL = 1e-5
GRAD_TOL = 1e-5       # of each gradient map's max |.|


def run(fx):
    out, ann, P2 = case_inputs(fx, "cuda")
    for t in out.values():
        t.requires_grad_(True)
    loss, stats = monoflex_loss.monoflex_head_loss(out, ann, P2)
    loss.backward()
    return loss, stats, {k: out[k].grad for k, _ in MAPS}


@pytest.mark.parametrize("case", CASES)
def test_terms_and_gradients_match_reference(case):
    fx = FX[case]
    loss, stats, grads = run(fx)
    assert set(stats) == set(TERMS) | {"total_loss"} and stats["total_loss"] is loss
    for i, key in enumerate(TERMS):
        got, ref = stats[key], float(fx["terms"][i])
        assert got.shape == () and got.dtype == torch.float32 and got.is_cuda
        assert abs(float(got.detach()) - ref) <= LOSS_RTOL * abs(ref), (key, float(got), ref)
        if case == "c" and key not in ("hm_loss", "hp_loss", "rot_loss"):
            assert float(got.detach()) == 0.0, key
    assert abs(float(loss.detach()) - float(fx["total"])) <= LOSS_RTOL * abs(float(fx["total"]))
    for name, _ in MAPS:
        g = grads[name].reshape(-1).cpu().numpy()
        idx, ref, gmax = fx[f"grad_{name}_idx"], fx[f"grad_{name}"], float(fx[f"grad_{name}_max"])
        if gmax == 0:
            assert not g.any(), name
            continue
        assert np.abs(g[idx] - ref).max() <= GRAD_TOL * gmax, (name, np.abs(g[idx] - ref).max(), gmax)
        assert abs(float(np.abs(g).max()) - gmax) <= GRAD_TOL * gmax, name
        if name != "hm":                                          # zero wherever the reference's is
            others = np.ones(g.size, dtype=bool)
            others[idx] = False
            assert not g[others].any(), name


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
        loss, _ = monoflex_loss.monoflex_head_loss(out, ann, P2)
        n_fwd = _lib.launch_count()
        loss.backward()
        assert n_fwd == 3 and _lib.launch_count() == 4            # hm, rows, combine; backward: one kernel


def test_cuda_graph_replay_bit_identical():
    out, ann, P2 = case_inputs(FX["b"], "cuda")
    for t in out.values():
        t.requires_grad_(True)

    def step():
        for t in out.values():
            t.grad = None
        loss, stats = monoflex_loss.monoflex_head_loss(out, ann, P2)
        loss.backward()
        return [loss] + [stats[k] for k in TERMS] + [out[k].grad for k, _ in MAPS]

    graph_replay_matches_eager(step)


def test_backward_of_a_single_term():
    """d hm_loss alone: only the heatmap gets a gradient, the same one the total gives it."""
    fx = FX["a"]
    _, _, grads = run(fx)
    out, ann, P2 = case_inputs(fx, "cuda")
    for t in out.values():
        t.requires_grad_(True)
    _, stats = monoflex_loss.monoflex_head_loss(out, ann, P2)
    stats["hm_loss"].backward()
    assert torch.equal(out["hm"].grad, grads["hm"])
    for k, _ in MAPS[1:]:
        assert not out[k].grad.any(), k


def test_ind_outside_the_map_gives_nan():
    fx = FX["b"]
    out, ann, P2 = case_inputs(fx, "cuda")
    H, W = int(fx["H"]), int(fx["W"])
    ann["ind"] = ann["ind"].clone()
    ann["ind"][1, 3] = H * W
    loss, stats = monoflex_loss.monoflex_head_loss(out, ann, P2)
    assert torch.isnan(loss).item() and all(torch.isnan(stats[k]).item() for k in TERMS)


def test_reference_head_training_step():
    out = run_seam_worker("monoflex_loss_step.py")
    assert out["native_bound"] and out["same_params"] and out["n_grads"] >= 36
    assert out["loss_rel_max"] <= LOSS_RTOL, out["loss_rel"]
    assert out["grad_err_max"] <= GRAD_TOL, out["grad_err_worst"]
