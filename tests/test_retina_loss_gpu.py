"""The native RetinaNet head loss on the GPU (csrc/retina_loss.cu through visualdet3d_b200/retina_loss.py) against the unmodified
reference loss (tests/golden/make_golden_retina_loss.py): assignment and counts bit-exact, 0-d losses within 1e-5 relative, gradients
within 1e-5 of each tensor's max |.| (plus the reference's own one-ulp spread where decoded boxes barely overlap) with the
reference's exact zeros, the same bits at an odd annotation row count, bit-identical reruns and CUDA-graph replays, a fixed launch count,
NaN for an out-of-range class, and reference training steps (head, and the whole detector) with the native loss installed."""
import numpy as np
import pytest
import torch

from loss_harness import graph_replay_matches_eager, run_seam_worker
from test_retina_loss_cpu import CASES, FX, case_inputs
from visualdet3d_b200 import _lib, retina_loss

pytestmark = pytest.mark.gpu
LOSS_RTOL = 1e-5
GRAD_TOL = 1e-5       # of each gradient tensor's max |.|


def run(fx):
    cls, reg, anchors, ann, cfg = case_inputs(fx, "cuda")
    cls.requires_grad_(True)
    reg.requires_grad_(True)
    c, r, d = retina_loss.retinanet_head_loss(cls, reg, anchors, ann, cfg)
    (c + r).backward()
    return c, r, d, cls.grad, reg.grad


@pytest.mark.parametrize("case", CASES)
def test_assignment_and_counts_bit_exact(case):
    fx = FX[case]
    cls, reg, anchors, ann, cfg = case_inputs(fx, "cuda")
    assign, counts = retina_loss.assignment(cls, reg, anchors, ann, cfg)
    assert assign.dtype == torch.int32 and counts.dtype == torch.int32
    assert np.array_equal(assign.cpu().numpy(), fx["assign"].astype(np.int32))
    assert np.array_equal(counts.cpu().numpy(), fx["counts"])


@pytest.mark.parametrize("case", CASES)
def test_losses_and_gradients_match_reference(case):
    fx = FX[case]
    c, r, d, gc, gr = run(fx)
    for got, key in ((c, "cls_loss"), (r, "reg_loss"), (d["cls_loss"], "cls_loss"), (d["reg_loss"], "reg_loss"),
                     (d["total_loss"], "total_loss")):
        ref = float(fx[key])
        assert got.shape == () and got.dtype == torch.float32
        assert abs(float(got.detach()) - ref) <= LOSS_RTOL * abs(ref), (key, float(got), ref)
    B, N, C = gc.shape
    gr = gr.reshape(B * N, 4).cpu().numpy()
    gc = gc.reshape(B * N, C).cpu().numpy()
    rows = fx["grad_reg_rows"]
    if len(rows):
        # plus, per element, the reference's own spread under a one-ulp change of its exp results: where the decoded boxes barely
        # overlap, the overlap width is a small difference of large coordinates and exp's last ulp decides its leading digits
        err = np.abs(gr[rows] - fx["grad_reg"])
        assert (err <= GRAD_TOL * float(fx["grad_reg_max"]) + 4 * fx["grad_reg_spread"]).all()
        well = fx["grad_reg_spread"] <= 1e-6 * float(fx["grad_reg_max"])           # the well-conditioned elements: the plain bound
        assert well.mean() > 0.95 and err[well].max() <= GRAD_TOL * float(fx["grad_reg_max"])
        assert abs(float(np.abs(gr).max()) - float(fx["grad_reg_max"])) <= GRAD_TOL * float(fx["grad_reg_max"])
    others = np.ones(B * N, dtype=bool)
    others[rows] = False
    assert not gr[others].any()                                   # exactly zero off the positives
    got = gc[fx["grad_cls_rows"]]
    ref = fx["grad_cls"]
    free = ~fx["cut"]                                             # elements at the 1e-5 cut may flip on a last-ulp difference
    assert np.abs(got - ref)[free].max() <= GRAD_TOL * float(fx["grad_cls_max"])
    assert np.array_equal(got[free] == 0, ref[free] == 0)         # the reference's exact zeros, and only those
    assert abs(float(np.abs(gc).max()) - float(fx["grad_cls_max"])) <= GRAD_TOL * float(fx["grad_cls_max"])


def odd_rows(ann):
    """The same valid rows in their order, packed into the smallest odd row count that holds them (padding after them): a trainer pads
    annotations to the batch's largest row count, which is as often odd as even."""
    valid = ann[:, :, 4] != -1
    M = int(valid.sum(1).max()) | 1
    out = torch.full((ann.shape[0], M, ann.shape[2]), -1.0, device=ann.device)
    for b in range(ann.shape[0]):
        out[b, :int(valid[b].sum())] = ann[b][valid[b]]
    return out


@pytest.mark.parametrize("case", CASES)
def test_odd_row_count_bit_identical(case):
    fx = FX[case]
    cls, reg, anchors, ann, cfg = case_inputs(fx, "cuda")
    odd = odd_rows(ann)
    assert odd.shape[1] % 2 == 1
    assign, counts = retina_loss.assignment(cls, reg, anchors, odd, cfg)
    assert np.array_equal(assign.cpu().numpy(), fx["assign"].astype(np.int32))
    assert np.array_equal(counts.cpu().numpy(), fx["counts"])
    outs = []
    for a in (ann, odd):
        c_, r_ = cls.clone().requires_grad_(True), reg.clone().requires_grad_(True)
        c, r, _ = retina_loss.retinanet_head_loss(c_, r_, anchors, a, cfg)
        (c + r).backward()
        outs.append((c, r, c_.grad, r_.grad))
    for x, y in zip(*outs):
        assert torch.equal(x, y)


def test_backward_through_one_term():
    cls, reg, anchors, ann, cfg = case_inputs(FX["edge"], "cuda")
    cls.requires_grad_(True)
    reg.requires_grad_(True)
    c, r, _ = retina_loss.retinanet_head_loss(cls, reg, anchors, ann, cfg)
    _, _, _, gc, gr = run(FX["edge"])
    (2.0 * r).backward()
    assert not cls.grad.any() and torch.allclose(reg.grad, 2.0 * gr, rtol=1e-6, atol=0)


def test_two_runs_bit_identical():
    a = run(FX["train"])
    b = run(FX["train"])
    for x, y in zip(a[:2] + a[3:], b[:2] + b[3:]):
        assert torch.equal(x, y)


def test_launch_count_fixed():
    cls, reg, anchors, ann, cfg = case_inputs(FX["train"], "cuda")
    cls.requires_grad_(True)
    _lib.launch_count_reset()
    c, r, _ = retina_loss.retinanet_head_loss(cls, reg, anchors, ann, cfg)
    n_fwd = _lib.launch_count()
    (c + r).backward()
    assert n_fwd == 3 and _lib.launch_count() == 4                 # iou_max, assign, combine (+ one memset); backward: one kernel


def test_cuda_graph_replay_bit_identical():
    cls, reg, anchors, ann, cfg = case_inputs(FX["edge"], "cuda")
    cls.requires_grad_(True)
    reg.requires_grad_(True)

    def step():
        cls.grad = reg.grad = None
        c, r, d = retina_loss.retinanet_head_loss(cls, reg, anchors, ann, cfg)
        (c + r).backward()
        return d["total_loss"], cls.grad, reg.grad

    graph_replay_matches_eager(step)


def test_out_of_range_class_gives_nan():
    cls, reg, anchors, ann, cfg = case_inputs(FX["edge"], "cuda")
    ann = ann.clone()
    valid = (ann[0, :, 4] != -1).nonzero()[0, 0]
    ann[0, valid, 4] = 3.0                                        # C = 3: one past the last class
    cls.requires_grad_(True)
    reg.requires_grad_(True)
    c, r, d = retina_loss.retinanet_head_loss(cls, reg, anchors, ann, cfg)
    (c + r).backward()
    torch.cuda.synchronize()
    assert torch.isnan(c) and torch.isnan(r) and torch.isnan(d["total_loss"])
    assert torch.isnan(cls.grad).all() and torch.isnan(reg.grad).all()


def test_no_positive_reg_loss_is_zero_tensor():
    c, r, d, gc, gr = run(FX["nopos"])
    assert r.shape == () and float(r.detach()) == 0.0 and float(FX["nopos"]["reg_loss"]) == 0.0
    assert not bool(FX["nopos"]["reg_loss_is_tensor"])           # the reference's is the Python number 0.0
    assert not gr.any()


def _worker(name, *args):
    out = run_seam_worker(name, *args)
    assert out["native_bound"] and out["same_params"] and out["n_grads"] > 1
    assert out["cls_rel"] <= LOSS_RTOL and out["reg_rel"] <= LOSS_RTOL and out["total_rel"] <= LOSS_RTOL
    assert out["grad_err_max"] <= GRAD_TOL, out["grad_err_worst"]
    return out


def test_reference_head_training_step():
    _worker("retina_loss_step.py", "head")


def test_reference_detector_training_step():
    out = _worker("retina_loss_step.py", "detector")
    assert out["n_grads"] > 100                                   # backbone, FPN and head parameters
