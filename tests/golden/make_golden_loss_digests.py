"""SHA-256 digests of every output of the five GPU training losses (anchor, RetinaNet, MonoFlex, KM3D, disparity) on every case of
their fixtures -> tests/golden/loss_digests.npz: losses, terms and totals, the anchor assignment and counts, and every gradient.  The
reference comparisons hold the losses to 1e-5, which a reordered sum passes; the digests pin the outputs bit for bit, so a change to how the
losses are organised (shared reductions, shared host code) must reproduce them exactly.  Needs a GPU:

    python tests/golden/make_golden_loss_digests.py

`tests/test_loss_digests_gpu.py` imports CASES, run_case and digest from here."""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.join(ROOT, "tests", "golden", "loss_digests.npz")
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

CASES = {"anchor": ["a", "b", "c"], "retina": ["train", "edge", "argmax", "nopos"], "monoflex": ["a", "b", "c"],
         "km3d": ["a", "b", "c", "d", "e"], "disparity": ["a", "b", "c", "d"]}


def _anchor(case):
    from test_anchor_loss_cpu import FX, case_inputs
    from visualdet3d_b200 import anchor_loss
    cls, reg, anchors, ann, loss_cfg = case_inputs(FX[case], "cuda")
    assign, counts = anchor_loss.assignment(cls, reg, anchors, ann, loss_cfg)
    cls.requires_grad_(True)
    reg.requires_grad_(True)
    c, r, d = anchor_loss.anchor3d_head_loss(cls, reg, anchors, ann, loss_cfg)
    (c + r).sum().backward()
    return dict(cls_loss=c, reg_loss=r, total_loss=d["total_loss"], assign=assign, counts=counts, grad_cls=cls.grad, grad_reg=reg.grad)


def _retina(case):
    from test_retina_loss_cpu import FX, case_inputs
    from visualdet3d_b200 import retina_loss
    cls, reg, anchors, ann, cfg = case_inputs(FX[case], "cuda")
    assign, counts = retina_loss.assignment(cls, reg, anchors, ann, cfg)
    cls.requires_grad_(True)
    reg.requires_grad_(True)
    c, r, d = retina_loss.retinanet_head_loss(cls, reg, anchors, ann, cfg)
    (c + r).backward()
    return dict(cls_loss=c, reg_loss=r, total_loss=d["total_loss"], assign=assign, counts=counts, grad_cls=cls.grad, grad_reg=reg.grad)


def _maps_loss(out, loss, stats, maps):
    got = {f"stat_{k}": v for k, v in stats.items()}
    got["loss"] = loss
    got.update({f"grad_{k}": out[k].grad for k, _ in maps})
    return got


def _monoflex(case):
    from test_monoflex_loss_cpu import FX, case_inputs
    from visualdet3d_b200 import monoflex_loss
    out, ann, P2 = case_inputs(FX[case], "cuda")
    for t in out.values():
        t.requires_grad_(True)
    loss, stats = monoflex_loss.monoflex_head_loss(out, ann, P2)
    loss.backward()
    return _maps_loss(out, loss, stats, monoflex_loss.MAPS)


def _km3d(case):
    from test_km3d_loss_cpu import FX, GEN, case_inputs
    from visualdet3d_b200 import km3d_loss
    fx = FX[case]
    out, ann, P2 = case_inputs(fx, "cuda")
    for t in out.values():
        t.requires_grad_(True)
    cfg = km3d_loss.LossConfig(output_w=float(fx["W"]), rampup_length=float(GEN.RAMPUP))
    loss, stats = km3d_loss.km3d_head_loss(out, ann, P2, GEN.GRAD_EPOCH, cfg)
    loss.backward()
    return _maps_loss(out, loss, stats, km3d_loss.MAPS)


def _disparity(case):
    from test_disparity_loss_cpu import FX, GEN
    from visualdet3d_b200 import disparity_loss
    x, label = GEN.inputs(case)
    x = x.cuda().requires_grad_(True)
    loss = disparity_loss.disparity_loss(x, label.cuda(), int(FX[case]["max_disp"]))
    loss.backward()
    return dict(loss=loss, grad=x.grad)


_RUN = dict(anchor=_anchor, retina=_retina, monoflex=_monoflex, km3d=_km3d, disparity=_disparity)


def run_case(loss, case):
    """-> {key: output array} of one fixture case of one loss"""
    import torch
    got = _RUN[loss](case)
    torch.cuda.synchronize()
    return {k: v.detach().cpu().numpy() for k, v in got.items()}


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main():
    fx = {}
    for loss, cases in CASES.items():
        for case in cases:
            for key, a in run_case(loss, case).items():
                fx[f"{loss}/{case}/{key}"] = np.array(digest(a))
                print(loss, case, key, a.dtype, a.shape, fx[f"{loss}/{case}/{key}"], flush=True)
    np.savez(OUT, **fx)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
