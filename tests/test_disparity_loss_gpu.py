"""The native disparity loss on the GPU (csrc/disparity_loss.cu through visualdet3d_b200/disparity_loss.py) against the unmodified
reference loss (tests/golden/make_golden_disparity_loss.py): the loss within 1e-5 relative, the gradient within 1e-5 of its max |.| at the
stored positions (the band and edge pixels included) and exactly zero outside the loss mask, bit-identical reruns and CUDA-graph replays,
the launch counts, no volume-sized allocation in the forward, and a reference Stereo3D training step with the native losses installed."""
import numpy as np
import pytest
import torch

from loss_harness import graph_replay_matches_eager, run_seam_worker
from test_disparity_loss_cpu import CASES, FX, GEN
from visualdet3d_b200 import _lib, disparity_loss

pytestmark = pytest.mark.gpu
LOSS_RTOL = 1e-5
GRAD_TOL = 1e-5       # of the gradient's max |.|


def case_inputs(case):
    x, label = GEN.inputs(case)
    return x.cuda().requires_grad_(True), label.cuda()


def run(case, scale=1.0):
    x, label = case_inputs(case)
    loss = disparity_loss.disparity_loss(x, label, int(FX[case]["max_disp"]))
    (loss * scale).backward()
    return loss, x.grad, label


@pytest.mark.parametrize("case", CASES)
def test_loss_and_gradient_match_reference(case):
    fx = FX[case]
    loss, grad, label = run(case)
    assert loss.shape == () and loss.dtype == torch.float32
    ref = float(fx["loss"])
    assert abs(float(loss) - ref) <= LOSS_RTOL * abs(ref), (float(loss), ref)
    gmax = float(fx["grad_max"])
    g = grad.reshape(-1)[torch.from_numpy(fx["grad_idx"]).cuda()].cpu().numpy()
    assert np.abs(g - fx["grad"]).max() <= GRAD_TOL * gmax
    assert abs(float(grad.abs().max()) - gmax) <= GRAD_TOL * gmax
    D = int(fx["max_disp"])
    outside = ~((label > 0) & (label < D))
    assert not grad.permute(1, 0, 2, 3)[:, outside].any()                    # exact zeros outside the loss mask


def test_no_valid_pixel_gives_exact_zeros():
    loss, grad, _ = run("c")
    assert float(loss) == 0.0 and not grad.any()


def test_non_finite_label_gives_nan():
    x, label = case_inputs("b")
    for bad in (float("nan"), float("inf")):
        lab = label.clone()
        lab[2, 3, 3] = bad
        assert torch.isnan(disparity_loss.disparity_loss(x, lab)).item()


def test_offset_logits_cancel_nothing():
    """+1000 on every logit of the training-shape volume leaves the loss and gradient (a shift-invariant function) where they were."""
    x, label = case_inputs("a")
    base = disparity_loss.disparity_loss(x, label)
    x2 = (x.detach() + 1000.0).requires_grad_(True)
    shifted = disparity_loss.disparity_loss(x2, label)
    assert abs(float(shifted) - float(base)) <= 1e-4 * abs(float(base))


def test_two_runs_bit_identical():
    a = run("a")
    b = run("a")
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_grad_output_scales_the_gradient():
    l1, g1, _ = run("d")
    l2, g2, _ = run("d", scale=0.37)
    assert torch.equal(l1, l2)
    assert float((g2 - 0.37 * g1).abs().max()) <= 1e-6 * float(g1.abs().max())


def test_launch_counts_fixed():
    x, label = case_inputs("a")
    _lib.launch_count_reset()
    loss = disparity_loss.disparity_loss(x, label)
    assert _lib.launch_count() == 2                                          # per-pixel pass, combine
    loss.backward()
    assert _lib.launch_count() == 3                                          # backward: one kernel


def test_forward_allocates_nothing_volume_sized():
    x, label = case_inputs("a")
    B, D, H, W = x.shape
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    loss = disparity_loss.disparity_loss(x, label)
    torch.cuda.synchronize()
    ws = int(_lib.load().vd3d_disparity_loss_workspace_bytes(B, D, H, W))
    bound = B * H * W * 4 + ws + 4096                                        # lse, the block partials, the loss (512-byte blocks)
    assert torch.cuda.max_memory_allocated() - before <= bound
    del loss


def test_cuda_graph_replay_bit_identical():
    x, label = case_inputs("b")

    def step():
        x.grad = None
        loss = disparity_loss.disparity_loss(x, label)
        loss.backward()
        return loss, x.grad

    graph_replay_matches_eager(step)


def test_reference_stereo3d_training_step():
    out = run_seam_worker("stereo3d_loss_step.py", timeout=1200)
    assert out["native_bound"] and out["same_params"] and out["disp_loss_ran"]
    assert out["cls_rel"] <= LOSS_RTOL and out["reg_rel"] <= LOSS_RTOL and out["disp_rel"] <= LOSS_RTOL
    assert out["depth_grad_err"] <= GRAD_TOL, out["depth_grad_worst"]
    assert out["head_grad_err"] <= GRAD_TOL, out["head_grad_worst"]
    assert out["trunk_grad_err"] <= 1e-4, out["trunk_grad_worst"]
