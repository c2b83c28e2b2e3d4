"""The native 3-D anchor head loss on the GPU (csrc/anchor_loss.cu through visualdet3d_b200/anchor_loss.py) against the unmodified
reference loss (tests/golden/make_golden_anchor_loss.py): assignment and counts bit-exact, losses within 1e-5 relative, gradients within
1e-5 of each tensor's max |.|, bit-identical reruns and CUDA-graph replays, and a reference StereoHead training step with the native
loss installed."""
import numpy as np
import pytest
import torch

from loss_harness import graph_replay_matches_eager, run_seam_worker
from test_anchor_loss_cpu import CASES, FX, case_inputs
from visualdet3d_b200 import _lib, anchor_loss

pytestmark = pytest.mark.gpu
LOSS_RTOL = 1e-5
GRAD_TOL = 1e-5       # of each gradient tensor's max |.|


def run(fx):
    cls, reg, anchors, ann, loss_cfg = case_inputs(fx, "cuda")
    cls.requires_grad_(True)
    reg.requires_grad_(True)
    c, r, d = anchor_loss.anchor3d_head_loss(cls, reg, anchors, ann, loss_cfg)
    (c + r).sum().backward()
    return c, r, d, cls.grad, reg.grad


@pytest.mark.parametrize("case", CASES)
def test_assignment_and_counts_bit_exact(case):
    fx = FX[case]
    cls, reg, anchors, ann, loss_cfg = case_inputs(fx, "cuda")
    assign, counts = anchor_loss.assignment(cls, reg, anchors, ann, loss_cfg)
    assert np.array_equal(assign.cpu().numpy(), fx["assign"])
    assert np.array_equal(counts.cpu().numpy(), fx["counts"])


@pytest.mark.parametrize("case", CASES)
def test_losses_and_gradients_match_reference(case):
    fx = FX[case]
    c, r, d, gc, gr = run(fx)
    for got, key in ((c, "cls_loss"), (r, "reg_loss"), (d["cls_loss"], "cls_loss"), (d["reg_loss"], "reg_loss"),
                     (d["total_loss"], "total_loss")):
        ref = fx[key].astype(np.float64)
        assert got.shape == (1,) and got.dtype == torch.float32
        assert abs(float(got.detach()) - float(ref[0])) <= LOSS_RTOL * abs(float(ref[0])), (key, float(got), float(ref[0]))
    B, N, C1 = gc.shape
    gr = gr.reshape(B * N, 12).cpu().numpy()
    gc = gc.reshape(B * N, C1).cpu().numpy()
    rows = fx["grad_reg_rows"]
    assert np.abs(gr[rows] - fx["grad_reg"]).max() <= GRAD_TOL * float(fx["grad_reg_max"])
    others = np.ones(B * N, dtype=bool)
    others[rows] = False
    assert not gr[others].any()                                  # zero wherever the reference's is
    assert np.abs(gc[fx["grad_cls_rows"]] - fx["grad_cls"]).max() <= GRAD_TOL * float(fx["grad_cls_max"])
    assert abs(float(np.abs(gc).max()) - float(fx["grad_cls_max"])) <= GRAD_TOL * float(fx["grad_cls_max"])
    assert not gc[fx["assign"].reshape(-1) == -2].any()          # nothing outside the mask


def test_two_runs_bit_identical():
    a = run(FX["a"])
    b = run(FX["a"])
    for x, y in zip(a[:2] + a[3:], b[:2] + b[3:]):
        assert torch.equal(x, y)


def test_launch_count_fixed():
    fx = FX["a"]
    cls, reg, anchors, ann, loss_cfg = case_inputs(fx, "cuda")
    cls.requires_grad_(True)
    _lib.launch_count_reset()
    c, r, _ = anchor_loss.anchor3d_head_loss(cls, reg, anchors, ann, loss_cfg)
    n_fwd = _lib.launch_count()
    (c + r).sum().backward()
    assert n_fwd == 3 and _lib.launch_count() == 4                 # iou_max, assign, combine (+ one memset); backward: one kernel


def test_cuda_graph_replay_bit_identical():
    fx = FX["c"]
    cls, reg, anchors, ann, loss_cfg = case_inputs(fx, "cuda")
    cfg = anchor_loss.LossConfig.from_loss_cfg(loss_cfg, cls.shape[-1] - 1)
    cls.requires_grad_(True)
    reg.requires_grad_(True)

    def step():
        cls.grad = reg.grad = None
        c, r, d = anchor_loss.anchor3d_head_loss(cls, reg, anchors, ann, cfg)
        (c + r).sum().backward()
        return d["total_loss"], cls.grad, reg.grad

    graph_replay_matches_eager(step)


def test_reference_head_training_step():
    out = run_seam_worker("anchor_loss_step.py")
    assert out["native_bound"] and out["same_params"] and out["n_grads"] > 10
    assert out["cls_rel"] <= LOSS_RTOL and out["reg_rel"] <= LOSS_RTOL and out["total_rel"] <= LOSS_RTOL
    assert out["grad_err_max"] <= GRAD_TOL, out["grad_err_worst"]
    assert all(n.endswith(".bias") for n in out["noise_floor_tensors"])          # only biases ahead of a BatchNorm
