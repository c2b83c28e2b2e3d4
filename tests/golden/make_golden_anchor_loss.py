"""Golden vectors for visualdet3d_b200/anchor_loss.py from the UNMODIFIED reference head loss (R/networks/heads/detection_3d_head.py:
402-498) run on the host through oracle/refload.py.
python tests/golden/make_golden_anchor_loss.py  ->  tests/golden/anchor_loss.npz

Cases (synthetic priors of `synth.synth_priors`, with its invalid-sentinel cells; head outputs of `synth.synth_head_outputs`):
  a  Stereo3D_example head (StereoHead: 2 classes, balance [20, 40], match_low_quality), B=4 at 288x1280 (N = 69120); image 1 has a
     padding row between ground truths
  b  Yolo3D_example head (1 class, match_low_quality=False), B=2 at 288x1280 (N = 46080)
  c  edge batch, Stereo3D head at 144x640 with every Pedestrian prior cell invalid: a normal image, an image without ground truth, an
     image of Pedestrians only (every positive dropped by the prior's z_mean > 0 selection) and an image with a ground truth that
     overlaps no masked anchor (zero max IoU: every zero-IoU anchor is assigned to it) between two others
Images are redrawn while any IoU lies within 1e-6 of 0.4 / 0.5 and, in a and b, while a ground truth overlaps no masked anchor; in b
also while a ground truth's max IoU is reached by two anchors.

The head outputs are regenerated from their seed by the tests, and the anchors / priors by `anchors.AnchorTable` (their sha256 is
stored and checked), so the file holds: annotations, P2, the priors, the mask (packed bits), the three losses, each image's
assigned_gt_inds over all N anchors (-2 outside the mask, -1 for an image without ground truth) and counts (positives assigned,
positives kept by the prior, negatives), captured by wrapping `_assign` / `_get_anchor_3d`, and the gradients of cls_loss + reg_loss:
grad_reg at every anchor where it is non-zero, grad_cls at every positive anchor and a strided sample of the rest, and each gradient's
max |.| over the whole tensor.
"""
import hashlib
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, ROOT)
import refload  # noqa: E402
from visualdet3d_b200 import synth  # noqa: E402

CASES = {
    "a": dict(kind="Stereo3D", B=4, H=288, W=1280, seed=11, n_gt=(2, 6), pad_middle=1),
    "b": dict(kind="Yolo3D", B=2, H=288, W=1280, seed=12, n_gt=(2, 5), pad_middle=-1),
    "c": dict(kind="edge", B=4, H=144, W=640, seed=13, n_gt=(2, 4), pad_middle=-1),
}
M_ROWS = 8
CLS_SAMPLE_STRIDE = 53


def sha(t: torch.Tensor) -> str:
    return hashlib.sha256(np.ascontiguousarray(t.detach().cpu().numpy().astype(np.float32)).tobytes()).hexdigest()


def head_setup(kind: str, preprocessed_path: str):
    """(obj_types, head cfg dict) of a case; the same on the host and in the tests."""
    if kind == "Yolo3D":
        return ["Car"], synth.mono3d_cfg(preprocessed_path, "GroundAwareYolo3D").head
    return ["Car", "Pedestrian"], synth.stereo3d_cfg(preprocessed_path).head


def case_priors(kind: str):
    obj_types = ["Car"] if kind == "Yolo3D" else ["Car", "Pedestrian"]
    n_ratios = 2 if kind == "Yolo3D" else 3
    pm, ps = synth.synth_priors(16, n_ratios, obj_types)
    if kind == "edge":                          # every Pedestrian cell invalid: an image of Pedestrians keeps no positive
        pm[1], ps[1] = -100.0, 1e10
    return pm, ps


def calc_iou(a, b):
    from visualDet3D.networks.utils.utils import calc_iou as ref_calc_iou
    return ref_calc_iou(a, b)


def draw_gt(rng, C, H, W, cls=None):
    w = rng.uniform(24, min(320, W * 0.5))
    h = min(w * rng.uniform(0.4, 1.3), H * 0.7)
    x1 = rng.uniform(0, W - w)
    y1 = rng.uniform(H * 0.35, H - h) if H - h > H * 0.35 else rng.uniform(0, H - h)
    c = rng.randint(C) if cls is None else cls
    z = rng.uniform(5, 50)
    return [x1, y1, x1 + w, y1 + h, c, x1 + w / 2 + rng.uniform(-6, 6), y1 + h / 2 + rng.uniform(-6, 6), z,
            rng.uniform(1.4, 1.9), rng.uniform(1.3, 1.7), rng.uniform(3.2, 4.6), rng.uniform(-np.pi, np.pi)]


def ok_image(rows, anchors_m, need_overlap: bool, no_ties: bool, zero_row=None) -> bool:
    if not rows:
        return True
    gt = torch.tensor(np.array(rows, dtype=np.float32))
    iou = calc_iou(anchors_m, gt[:, :4])
    for thr in (0.4, 0.5):
        if ((iou - thr).abs() < 1e-6).any():
            return False
    gmax = iou.max(dim=0).values
    for i in range(len(rows)):
        if i == zero_row:
            if gmax[i] != 0:
                return False
            continue
        if need_overlap and not gmax[i] > 0:
            return False
        if no_ties and int((iou[:, i] == gmax[i]).sum()) > 1:
            return False
    return True


def draw_annotations(case, C, anchors, mask):
    """[B, M_ROWS, 12] compound_annotation rows, -1 padding."""
    rng = np.random.RandomState(case["seed"])
    B, H, W = case["B"], case["H"], case["W"]
    ann = np.full((B, M_ROWS, 12), -1.0, dtype=np.float32)
    for b in range(B):
        am = anchors[mask[b]]
        for _ in range(1000):
            zero_row, cls = None, None
            if case["kind"] == "edge" and b == 1:
                rows = []
            else:
                n = rng.randint(case["n_gt"][0], case["n_gt"][1] + 1)
                if case["kind"] == "edge" and b == 2:
                    cls = 1
                rows = [draw_gt(rng, C, H, W, cls if cls is not None else (0 if case["kind"] == "edge" else None)) for _ in range(n)]
                if case["kind"] == "edge" and b == 3:
                    # a small box that overlaps masked-out anchors only (masked anchors of every scale cover the whole image, so it
                    # lies below the image, where only the tallest anchors reach), between two ordinary ground truths
                    zero_row = 1
                    au = anchors[~mask[b]]
                    free = []
                    for y in range(H, 3 * H, 4):
                        for x in range(0, W - 12, 32):
                            box = torch.tensor([[x, y, x + 10.0, y + 6.0]])
                            if float(calc_iou(am, box).max()) == 0.0 and float(calc_iou(au, box).max()) > 0.0:
                                free.append((x, y))
                    x, y = free[rng.randint(len(free))]
                    zrow = draw_gt(rng, C, H, W, 0)
                    zrow[:4] = [x, y, x + 10.0, y + 6.0]
                    rows.insert(zero_row, zrow)
            if ok_image(rows, am, need_overlap=True, no_ties=case["kind"] == "Yolo3D", zero_row=zero_row):
                break
        else:
            raise RuntimeError(f"case {case}: image {b} could not be drawn")
        slots = list(range(len(rows)))
        if b == case["pad_middle"] and len(rows) >= 2:
            slots = [s if s < 1 else s + 1 for s in slots]          # row 1 stays padding
        for s, r in zip(slots, rows):
            ann[b, s] = r
    return ann


def build_head(kind, tmp):
    import visualDet3D.networks  # noqa: F401  registers the detectors
    from visualDet3D.networks.heads.detection_3d_head import AnchorBasedDetection3DHead, StereoHead
    obj_types, hc = head_setup(kind, tmp)
    pm, ps = case_priors(kind)
    synth.write_priors(tmp, pm, ps, obj_types)
    layer = dict(num_features_in=8, num_cls_output=len(obj_types) + 1, num_reg_output=12, cls_feature_size=8, reg_feature_size=8)
    cls = AnchorBasedDetection3DHead if kind == "Yolo3D" else StereoHead
    head = cls(num_features_in=8, num_classes=len(obj_types), num_regression_loss_terms=13, preprocessed_path=tmp,
               anchors_cfg=refload.to_edict(dict(hc.anchors_cfg)), layer_cfg=refload.to_edict(layer),
               loss_cfg=refload.to_edict(dict(hc.loss_cfg)), test_cfg=refload.to_edict(dict(hc.test_cfg)))
    head.train()
    return head, obj_types, pm, ps


def run_case(name, case):
    tmp = tempfile.mkdtemp()
    head, obj_types, pm, ps = build_head(case["kind"], tmp)
    C = len(obj_types)
    B, H, W = case["B"], case["H"], case["W"]
    P2, _ = synth.synth_P2(B, H, W)
    anchors = head.get_anchor(torch.zeros(B, 3, H, W), P2)
    N = anchors["anchors"].shape[1]
    mask = anchors["mask"]
    ann = draw_annotations(case, C, anchors["anchors"][0], mask)
    cls_scores, reg_preds = synth.synth_head_outputs(B, N, C, seed=case["seed"])
    cls_scores.requires_grad_(True)
    reg_preds.requires_grad_(True)

    assigned, nsel = [], []
    orig_assign, orig_sel = head._assign, head._get_anchor_3d

    def cap_assign(*a, **k):
        r = orig_assign(*a, **k)
        assigned.append(r["assigned_gt_inds"].clone())
        return r

    def cap_sel(*a, **k):
        r = orig_sel(*a, **k)
        nsel[-1] = int(r[0].sum())
        return r

    head._assign, head._get_anchor_3d = cap_assign, cap_sel
    # nsel: one slot per image with ground truth, filled when _get_anchor_3d runs (it does not without positives)
    orig_sample = head._sample

    def cap_sample(*a, **k):
        nsel.append(0)
        return orig_sample(*a, **k)

    head._sample = cap_sample
    cls_loss, reg_loss, d = head.loss(cls_scores, reg_preds, anchors, torch.from_numpy(ann), P2)
    (cls_loss + reg_loss).sum().backward()

    assign = np.full((B, N), -2, dtype=np.int32)
    counts = np.zeros((B, 3), dtype=np.int32)
    it = iter(zip(assigned, nsel))
    for b in range(B):
        m = mask[b].numpy()
        if (ann[b, :, 4] != -1).sum() == 0:
            assign[b, m] = -1
            continue
        a, ns = next(it)
        a = a.numpy()
        assign[b, m] = a
        counts[b] = [(a > 0).sum(), ns, (a == 0).sum()]
    gc = cls_scores.grad.numpy()
    gr = reg_preds.grad.numpy()
    rows = np.nonzero(np.abs(gr.reshape(B * N, 12)).sum(1) > 0)[0]
    pos = np.nonzero(assign.reshape(-1) > 0)[0]
    flat = np.arange(B * N)
    cls_rows = np.union1d(pos, flat[::CLS_SAMPLE_STRIDE])
    from visualdet3d_b200.anchors import AnchorTable
    table = AnchorTable((H, W), head_setup(case["kind"], tmp)[1].anchors_cfg, pm, ps, "cpu")
    assert sha(table.anchors) == sha(anchors["anchors"][0]) and sha(table.mean_std) == sha(anchors["anchor_mean_std_3d"])
    out = dict(kind=np.array(case["kind"]), B=B, H=H, W=W, seed=case["seed"], pm=pm, ps=ps, P2=P2.numpy(), ann=ann,
               mask_bits=np.packbits(mask.numpy().reshape(-1)), anchors_sha=np.array(sha(anchors["anchors"][0])),
               mean_std_sha=np.array(sha(anchors["anchor_mean_std_3d"])),
               cls_loss=cls_loss.detach().numpy(), reg_loss=reg_loss.detach().numpy(), total_loss=d["total_loss"].detach().numpy(),
               assign=assign, counts=counts, grad_reg_rows=rows.astype(np.int64), grad_reg=gr.reshape(B * N, 12)[rows],
               grad_reg_max=np.float32(np.abs(gr).max()), grad_cls_rows=cls_rows.astype(np.int64),
               grad_cls=gc.reshape(B * N, C + 1)[cls_rows], grad_cls_max=np.float32(np.abs(gc).max()))
    print(f"case {name}: N={N} cls={float(cls_loss):.6g} reg={float(reg_loss):.6g} counts={counts.tolist()} "
          f"reg rows={len(rows)} cls rows={len(cls_rows)}")
    return out


def main():
    refload.load_reference()
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    fix = {}
    for name, case in CASES.items():
        for k, v in run_case(name, case).items():
            fix[f"{name}/{k}"] = v
    path = os.path.join(HERE, "anchor_loss.npz")
    np.savez_compressed(path, **fix)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
