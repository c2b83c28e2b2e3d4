"""Golden vectors of the RetinaNet 2-D detector: runs the UNMODIFIED reference (R/detectors/retinanet_2d.py, CPU, fp32) on the seeded
synthetic weights / inputs of visualdet3d_b200.synth and writes

    retinanet_96x320.npz        (B = 2; also the FULL cls / reg predictions and the reference's top-k / NMS indices, for the decode test)
    retinanet_288x1280.npz      (B = 1, the example config's shape)
    retinanet_64x128_nopre.npz  (B = 2, nms_pre = 0: the branch without top-k)
    retinanet_keys.json         (state_dict keys and shapes of the reference's RetinaNet)

    python tests/golden/make_golden_retinanet.py

The outputs must not depend on knife edges, so for every image the generator asserts (and stores in `margins`) that the top nms_pre + 1
scores are distinct, that the score at rank nms_pre is below score_thr (a boundary flip cannot change the output), that no candidate
score lies within 1e-4 of score_thr and that no IoU between two candidates above score_thr lies within 1e-4 of nms_iou_thr.  Otherwise it redraws the input
seed.
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import refload  # noqa: E402
from make_golden import flatten_fixture, subsample  # noqa: E402
from visualdet3d_b200 import synth  # noqa: E402

EPS = 1e-4


def iou_matrix(bx: torch.Tensor) -> torch.Tensor:
    """fp32 IoU with torchvision's CPU nms arithmetic (area = (x2 - x1) * (y2 - y1), inter / (a_i + a_j - inter))."""
    x1, y1, x2, y2 = bx.unbind(1)
    area = (x2 - x1) * (y2 - y1)
    w = (torch.minimum(x2[:, None], x2[None]) - torch.maximum(x1[:, None], x1[None])).clamp(min=0)
    h = (torch.minimum(y2[:, None], y2[None]) - torch.maximum(y1[:, None], y1[None])).clamp(min=0)
    inter = w * h
    return inter / (area[:, None] + area[None] - inter)


def margins(head, cls, reg, anchors, nms_pre, score_thr, iou_thr):
    """(top-k distinctness gap, score_thr - score at rank nms_pre, candidate score gap to score_thr, IoU gap to iou_thr) of one image,
    plus the reference's top-k indices (None without top-k) and its NMS keep indices into the candidate list."""
    p = cls.sigmoid()
    ms, _ = p.max(dim=-1)
    N = ms.shape[0]
    topk = None
    if nms_pre > 0 and N > nms_pre:
        s = torch.sort(ms, descending=True).values
        gap = float((s[:nms_pre] - s[1:nms_pre + 1]).min())
        rank_gap = float(score_thr - s[nms_pre])
        _, topk = ms.topk(nms_pre)
        cand = ms[topk]
        boxes = head._decode(anchors[topk], reg[topk])
    else:
        gap, rank_gap = float("inf"), float("inf")
        cand = ms
        boxes = head._decode(anchors, reg)
    score_gap = float((cand - score_thr).abs().min())
    # the output (rows above score_thr) depends only on the IoUs among the candidates above score_thr: a lower-scored box never
    # suppresses a higher-scored one, and whether a box below the threshold is kept changes no row of the output
    hi = cand > score_thr
    iou = iou_matrix(boxes[hi])
    iou.fill_diagonal_(-1.0)
    iou_gap = float((iou.double() - iou_thr).abs().min()) if int(hi.sum()) > 1 else float("inf")
    from torchvision.ops import nms
    keep = nms(boxes, cand, iou_thr)
    return (gap, rank_gap, score_gap, iou_gap), topk, keep


def gen(H, W, B, tag, nms_pre=1000, full=False, wseed=0):
    refload.load_reference()
    from visualDet3D.networks.utils.registry import DETECTOR_DICT
    cfg = synth.retinanet_cfg(nms_pre=nms_pre)
    model = DETECTOR_DICT["RetinaNet"](refload.to_edict(cfg))
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    with open(os.path.join(HERE, "retinanet_keys.json"), "w") as f:
        json.dump({k: list(v) for k, v in shapes.items()}, f, indent=0)
    sd = synth.synth_state_dict(shapes, wseed)
    res = model.load_state_dict(sd, strict=False)
    assert res.unexpected_keys == [] and all(k.endswith("balance_weights") for k in res.missing_keys), res
    model.eval()
    head = model.bbox_head
    tc = cfg.head.test_cfg
    for iseed in range(1, 200):
        img, _ = synth.synth_mono_inputs(B, H, W, seed=iseed)
        stages = {}
        hooks = [model.core.register_forward_hook(lambda m, i, o: stages.setdefault("P", []).append([t.detach().clone() for t in o])),
                 head.register_forward_hook(lambda m, i, o: stages.setdefault("head", []).append(o))]
        outs = []
        with torch.no_grad():
            for b in range(B):                      # the reference asserts batch 1 (retinanet_2d.py:134)
                outs.append(model([img[b:b + 1], None]))
        for h in hooks:
            h.remove()
        anchors = head.anchors.anchors[0]
        cls = torch.cat([x[0] for x in stages["head"]], 0)
        reg = torch.cat([x[1] for x in stages["head"]], 0)
        ok, per = True, []
        with torch.no_grad():
            for b in range(B):
                m, topk, keep = margins(head, cls[b], reg[b], anchors, nms_pre, tc.score_thr, tc.nms_iou_thr)
                per.append((m, topk, keep))
                ok = ok and m[0] > 0 and m[1] > EPS and m[2] > EPS and m[3] > EPS
        print(tag, "input seed", iseed, "margins", [p[0] for p in per], "detections", [len(o[0]) for o in outs])
        if ok:
            break
    else:
        raise RuntimeError("no input seed with clear margins")
    fix = {"meta": np.array([H, W, B, wseed, iseed, nms_pre], dtype=np.int64),
           "margins": np.array([p[0] for p in per], dtype=np.float64)}
    for b in range(B):
        s, bb, ci = outs[b]
        fix[f"scores_{b}"], fix[f"bboxes_{b}"], fix[f"cls_{b}"] = s.numpy(), bb.numpy(), ci.numpy()
        if full:
            m, topk, keep = per[b]
            fix[f"topk_{b}"] = (topk if topk is not None else torch.arange(cls.shape[1])).numpy().astype(np.int64)
            fix[f"keep_{b}"] = keep.numpy().astype(np.int64)
    for i in range(len(stages["P"][0])):
        fix[f"P{i}"] = subsample(torch.cat([x[i] for x in stages["P"]], 0))
    fix["cls_preds"], fix["reg_preds"] = subsample(cls), subsample(reg)
    fix["anchors"] = subsample(anchors)
    if full:
        fix["cls_full"], fix["reg_full"], fix["anchors_full"] = cls.numpy(), reg.numpy(), anchors.numpy()
    np.savez_compressed(os.path.join(HERE, tag + ".npz"), **flatten_fixture(fix))
    print("wrote", tag)


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    gen(96, 320, 2, "retinanet_96x320", full=True)
    gen(288, 1280, 1, "retinanet_288x1280")
    gen(64, 128, 2, "retinanet_64x128_nopre", nms_pre=0)
