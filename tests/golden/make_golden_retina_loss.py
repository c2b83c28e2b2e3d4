"""Golden vectors for visualdet3d_b200/retina_loss.py from the UNMODIFIED reference RetinaNet head loss (R/networks/heads/
retinanet_head.py:309-362) run on the host through oracle/refload.py.
python tests/golden/make_golden_retina_loss.py  ->  tests/golden/retina_loss.npz

Cases (RetinaNet_example anchors, 3 classes; head outputs of `synth.retina_head_outputs`; annotations in compound_annotation's 12 columns,
padding rows (class -1) interleaved between the valid ones):
  train    B=8 at 288x1280 (N = 69210), RetinaNet_example's head_loss (gamma 2, balance_weights [1], fg 0.5 / bg 0.4 / min 0), 2..12
           KITTI-like boxes per image
  edge     B=4 at 96x320, gamma 0, per-class balance weights, non-default target_means / target_stds: image 1 has no valid row; image 0
           has two rows with the same box and different classes (argmax takes the first, low-quality matching the last); image 2 has a
           16x16 box whose max IoU (0.25) is reached by several anchors, positive only through low-quality matching
  argmax   B=2 at 96x320, gt_max_assign_all=False (the single-anchor low-quality branch), with the tied 16x16 box
  nopos    B=2 at 96x320, match_low_quality=False and boxes too small to reach fg: no positive anywhere (the reference's reg_loss is then
           the Python number 0.0, stored as 0)

The head outputs are regenerated from their seed by the tests and the anchors by `anchors.grid_anchors` (their sha256 is stored and
checked), so the file holds: the loss settings, annotations, each image's assigned_gt_inds (int8, captured by wrapping `_assign`), the
counts (positives, negatives, ignored), the losses and the gradients of cls_loss + reg_loss: grad_reg at every positive, grad_cls at every
positive and a seeded sample of ~2000 other rows, each gradient's max |.| over the whole tensor, `cut` flags for the sampled cls
elements whose focal value before the 1e-5 cut lies within 1e-6 relative of it (a last-ulp difference in exp / log1p may flip those), and
grad_reg_spread: how far each positive's reg gradient moves under a one-ulp change of _decode's exp results (large only where the
decoded boxes barely overlap).
"""
import hashlib
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, ROOT)
import refload  # noqa: E402
from visualdet3d_b200 import synth  # noqa: E402

C = 3
M_ROWS = 16
N_SAMPLE = 2000
EXAMPLE_LOSS = dict(fg_iou_threshold=0.5, bg_iou_threshold=0.4, min_iou_threshold=0, gamma=2.0, balance_weights=[1], pos_weight=-1)
CASES = {
    "train": dict(B=8, H=288, W=1280, seed=21, n_gt=(2, 12), loss=EXAMPLE_LOSS),
    "edge": dict(B=4, H=96, W=320, seed=22, n_gt=(2, 4), loss=dict(EXAMPLE_LOSS, gamma=0.0, balance_weights=[0.5, 2.0, 4.0]),
                 means=[0.1, -0.05, 0.02, 0.0], stds=[0.2, 0.25, 0.5, 0.4]),
    "argmax": dict(B=2, H=96, W=320, seed=23, n_gt=(2, 3), loss=dict(EXAMPLE_LOSS, gt_max_assign_all=False)),
    "nopos": dict(B=2, H=96, W=320, seed=24, n_gt=(2, 4), loss=dict(EXAMPLE_LOSS, match_low_quality=False)),
}
TIED_BOX = [64.0, 28.0, 80.0, 44.0]        # inside the 32x32 level-3 anchors centred at x 68 / 76, y 28 / 36 / 44: IoU 0.25 each


def sha(t: torch.Tensor) -> str:
    return hashlib.sha256(np.ascontiguousarray(t.detach().cpu().numpy().astype(np.float32)).tobytes()).hexdigest()


def head_cfg(case):
    """cfg.detector.head of RetinaNet_example with the case's loss settings and targets (stacked_convs 0: the loss reads no feature)."""
    hc = synth.retinanet_cfg().head
    return refload.to_edict(dict(stacked_convs=0, in_channels=8, feat_channels=8, num_classes=C,
                                 target_stds=list(case.get("stds", hc.target_stds)), target_means=list(case.get("means", hc.target_means)),
                                 anchors_cfg=dict(hc.anchors_cfg), loss_cfg=dict(case["loss"]), test_cfg=dict(hc.test_cfg)))


def build_head(case):
    from visualDet3D.networks.heads.retinanet_head import RetinanetHead
    return RetinanetHead(**head_cfg(case)).train()


def row(rng, box, cls):
    """A compound_annotation row: the box and class the loss reads, then plausible 3-D columns it ignores."""
    x1, y1, x2, y2 = box
    return [x1, y1, x2, y2, cls, (x1 + x2) / 2, (y1 + y2) / 2, rng.uniform(5, 50), rng.uniform(1.4, 1.9), rng.uniform(1.3, 1.7),
            rng.uniform(3.2, 4.6), rng.uniform(-np.pi, np.pi)]


def kitti_box(rng, H, W, small=False):
    if small:
        w = rng.uniform(3, 7)
        h = w * rng.uniform(0.6, 1.4)
    else:
        w = rng.uniform(16, min(320, W * 0.5))
        h = min(w * rng.uniform(0.4, 1.3), H * 0.7)
    x1 = rng.uniform(0, W - w)
    y1 = rng.uniform(H * 0.35, H - h) if H - h > H * 0.35 else rng.uniform(0, H - h)
    return [x1, y1, x1 + w, y1 + h]


def draw_annotations(name, case):
    """[B, M_ROWS, 12], -1 padding, the valid rows scattered over the block in their order."""
    rng = np.random.RandomState(case["seed"])
    B, H, W = case["B"], case["H"], case["W"]
    ann = np.full((B, M_ROWS, 12), -1.0, dtype=np.float32)
    for b in range(B):
        n = rng.randint(case["n_gt"][0], case["n_gt"][1] + 1)
        rows = [row(rng, kitti_box(rng, H, W, small=name == "nopos"), rng.randint(C)) for _ in range(n)]
        if name == "edge" and b == 0:                      # the same box twice, different classes
            rows.insert(1, row(rng, rows[0][:4], (int(rows[0][4]) + 1) % C))
        if name == "edge" and b == 1:
            rows = []
        if (name == "edge" and b == 2) or name == "argmax":
            rows = [r for r in rows if r[0] > 140] + [row(rng, TIED_BOX, rng.randint(C))]
        slots = np.sort(rng.choice(M_ROWS, size=len(rows), replace=False))
        for s, r in zip(slots, rows):
            ann[b, s] = r
    return ann


def focal_before_cut(x, t, gamma, bw):
    """SigmoidFocalLoss's element value before the 1e-5 cut (losses.py:33-38), the reference's ops."""
    probs = torch.sigmoid(x)
    fw = torch.pow(torch.where(torch.eq(t, 1.0), 1.0 - probs, probs), gamma)
    bce = -(t * torch.nn.functional.logsigmoid(x)) * bw - ((1 - t) * torch.nn.functional.logsigmoid(-x))
    return fw * bce


def reg_grad_spread(head, anchors, gt, pred, scale):
    """[P, 4]: how far each positive's reg gradient moves when the four exp results of _decode (the prediction's and the target's dw, dh)
    are nudged by -1, 0 or +1 ulp.  Where the decoded boxes barely overlap, the overlap's width is a small difference of large
    coordinates, and a last-ulp difference in exp moves the gradient by far more than its rounding; this measures that conditioning.
    The reference's _encode and IoULoss, and its _decode's expression order with the exp results nudged."""
    means, stds = pred.new_tensor(head.target_means), pred.new_tensor(head.target_stds)
    target = head._encode(anchors, gt)

    def decode(d, nudge):
        dd = d * stds + means
        px, py = (anchors[:, 0] + anchors[:, 2]) * 0.5, (anchors[:, 1] + anchors[:, 3]) * 0.5
        pw, ph = anchors[:, 2] - anchors[:, 0], anchors[:, 3] - anchors[:, 1]
        e = [dd[:, k].exp() for k in (2, 3)]
        e = [x if s == 0 else x + (torch.nextafter(x, torch.full_like(x, s * np.inf)) - x).detach() for x, s in zip(e, nudge)]
        gw, gh, gx, gy = pw * e[0], ph * e[1], px + pw * dd[:, 0], py + ph * dd[:, 1]
        return torch.stack([gx - gw * 0.5, gy - gh * 0.5, gx + gw * 0.5, gy + gh * 0.5], dim=-1)

    grads = []
    for nudge in np.ndindex(3, 3, 3, 3):
        s = [v - 1 for v in nudge]
        p = pred.detach().clone().requires_grad_(True)
        head.loss_bbox(decode(p, s[:2]), decode(target, s[2:])).sum().backward()
        grads.append(p.grad * scale)
    g = torch.stack(grads)
    return (g - g[40]).abs().amax(0).numpy()                         # g[40]: no nudge


def run_case(name, case=None):
    case = case or CASES[name]
    torch.manual_seed(0)
    head = build_head(case)
    B, H, W = case["B"], case["H"], case["W"]
    anchors = head.get_anchor(torch.zeros(B, 3, H, W))
    N = anchors.shape[1]
    ann = draw_annotations(name, case)
    cls_scores, reg_preds = synth.retina_head_outputs(B, N, C, seed=case["seed"])
    cls_scores.requires_grad_(True)
    reg_preds.requires_grad_(True)

    assigned = []
    orig_assign = head._assign

    def cap_assign(*a, **k):
        r = orig_assign(*a, **k)
        assigned.append(r["assigned_gt_inds"].clone())
        return r

    head._assign = cap_assign
    cls_loss, reg_loss, d = head.loss(cls_scores, reg_preds, anchors, torch.from_numpy(ann))
    (cls_loss + reg_loss).backward()
    assign = torch.stack(assigned).numpy()
    assert assign.min() >= -1 and assign.max() < 127
    counts = np.stack([(assign > 0).sum(1), (assign == 0).sum(1), (assign == -1).sum(1)], axis=1).astype(np.int32)

    gc = cls_scores.grad.numpy().reshape(B * N, C)
    gr = (reg_preds.grad if reg_preds.grad is not None else torch.zeros_like(reg_preds)).numpy().reshape(B * N, 4)   # nopos: no graph
    flat = assign.reshape(-1)
    pos = np.nonzero(flat > 0)[0]
    rng = np.random.RandomState(case["seed"] + 1000)
    cls_rows = np.union1d(pos, rng.choice(B * N, size=N_SAMPLE, replace=False))
    # the sampled rows' targets (-1 ignored, 0, 1 at the positive's class) and focal values before the cut
    tgt = np.zeros((len(cls_rows), C), dtype=np.float32)
    a = flat[cls_rows]
    tgt[a < 0] = -1.0
    for i in np.nonzero(a > 0)[0]:
        b = cls_rows[i] // N
        valid = ann[b][ann[b, :, 4] != -1]
        tgt[i, int(valid[a[i] - 1, 4])] = 1.0
    bw = head.loss_cls.balance_weights
    f = focal_before_cut(cls_scores.detach().reshape(B * N, C)[torch.from_numpy(cls_rows)], torch.from_numpy(tgt), head.loss_cls.gamma, bw)
    cut = ((f - 1e-5).abs() <= 1e-6 * 1e-5).numpy() & (tgt != -1)
    pb, pn = np.divmod(pos, N)
    gt_rows = [ann[b][ann[b, :, 4] != -1][flat[f] - 1, :4] for b, f in zip(pb, pos)]
    spread = reg_grad_spread(head, anchors[0][torch.from_numpy(pn)], torch.from_numpy(np.array(gt_rows, dtype=np.float32).reshape(-1, 4)),
                             reg_preds.detach().reshape(B * N, 4)[torch.from_numpy(pos)], 1.0 / float(1e-4 + len(pos)))
    reg_value = reg_loss.detach().numpy() if torch.is_tensor(reg_loss) else np.array(reg_loss, dtype=np.float32)
    out = dict(B=B, H=H, W=W, seed=case["seed"], C=C, loss_cfg=np.array(json.dumps(case["loss"])),
               target_means=np.array(head.target_means, dtype=np.float64), target_stds=np.array(head.target_stds, dtype=np.float64),
               ann=ann, anchors_sha=np.array(sha(anchors[0])), assign=assign.astype(np.int8), counts=counts,
               cls_loss=cls_loss.detach().numpy(), reg_loss=reg_value, reg_loss_is_tensor=np.array(torch.is_tensor(reg_loss)),
               total_loss=np.asarray(d["total_loss"].detach().numpy()),
               grad_reg_rows=pos.astype(np.int64), grad_reg=gr[pos], grad_reg_max=np.float32(np.abs(gr).max()), grad_reg_spread=spread,
               grad_cls_rows=cls_rows.astype(np.int64), grad_cls=gc[cls_rows], grad_cls_max=np.float32(np.abs(gc).max()), cut=cut)
    print(f"case {name}: N={N} cls={float(cls_loss.detach()):.6g} reg={float(reg_value):.6g} counts={counts.tolist()} "
          f"cls rows={len(cls_rows)} cut flags={int(cut.sum())}")
    return out


def main():
    refload.load_reference()
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    fix = {}
    for name in CASES:
        for k, v in run_case(name).items():
            fix[f"{name}/{k}"] = v
    path = os.path.join(HERE, "retina_loss.npz")
    np.savez_compressed(path, **fix)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
