"""Constructed candidate sets for the device decode / sort / NMS stages (tests/test_decode_nms_edges_gpu.py), and CPU checks that each
builder produces what it claims: candidate counts, score ties, IoU values on the intended side of the threshold, plateau peaks, and a
host restatement of the RetinaNet decode that matches the reference's outputs.

Every case is exact in float32 by construction:
- boxes lie on a 0.5-pixel grid and the regression outputs are 0, so the decode reproduces the chosen boxes bit for bit;
- scores come from logits whose float32 sigmoid, 1 / (1 + exp(-x)) rounded step by step, does not depend on the last bits of exp(-x)
  (the result is the same for exp(-x) off by up to 4 ulp either way), so torch's CPU sigmoid and the device's agree bit for bit.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import torch_port as tp

F32 = np.float32
SCORE_THR_3D = 0.75          # the anchor heads' test_cfg.score_thr
NCLS_3D, T_3D = 2, 2         # classes (+1 alpha channel) and anchor types of the 3-D anchor head cases
CN_H, CN_W, CN_NCLS, CN_K = 24, 40, 3, 100


# ---------------------------------------------------------------------------------------------------------------------------------------
# exact scores
# ---------------------------------------------------------------------------------------------------------------------------------------
def sigmoid_f32(x):
    x = np.asarray(x, F32)
    with np.errstate(over="ignore"):
        e = np.exp(-x.astype(np.float64)).astype(F32)
    return (F32(1) / (F32(1) + e)).astype(F32)


def _robust(x):
    x = np.asarray(x, F32)
    e = np.exp(-x.astype(np.float64)).astype(F32)
    ref = F32(1) / (F32(1) + e)
    ok = np.ones(len(x), bool)
    for k in range(-4, 5):
        ek = (e.view(np.int32) + k).view(F32)
        ok &= (F32(1) / (F32(1) + ek)) == ref
    t = torch.from_numpy(x.copy())
    ok &= torch.sigmoid(t).numpy() == ref                                    # torch's vectorised path ...
    ok &= np.array([torch.sigmoid(t[i:i + 1]).item() for i in range(len(x))], F32) == ref    # ... and its scalar tail
    return ok


def logits_for(scores):
    """float32 logits whose sigmoid is exactly `scores` on the host and the device: scores in [0.97, 1) are inverted and searched
    ulp by ulp for a robust logit; 1.0 and 0.0 come from saturating logits (>= 17 and <= -104)."""
    s = np.asarray(scores, F32)
    out = np.zeros(len(s), F32)
    found = np.zeros(len(s), bool)
    out[s == 1], found[s == 1] = 20.0, True
    out[s == 0], found[s == 0] = -110.0, True
    mid = ~found
    assert bool(((s[mid] >= 0.97) & (s[mid] < 1)).all()), "exact scores lie in [0.97, 1), or are 0 or 1"
    with np.errstate(divide="ignore"):
        x0 = np.log(s.astype(np.float64) / (1 - s.astype(np.float64))).astype(F32)
    for k in sorted(range(-64, 65), key=abs):
        todo = ~found
        if not todo.any():
            break
        xk = (x0[todo].view(np.int32) + k).view(F32)
        ok = (sigmoid_f32(xk) == s[todo]) & _robust(xk)
        idx = np.nonzero(todo)[0][ok]
        out[idx], found[idx] = xk[ok], True
    assert found.all(), "no robust logit for some scores"
    return out


def sc(v):
    """the float32 sigmoid value nearest to v: a float32 sigmoid is 1 / fl(1 + e), and fl(1 + e) = 1 + k 2^-23 near 1, so only about
    every second float32 in [0.5, 1) is the sigmoid of some float32"""
    v = np.asarray(v, np.float64)
    k = np.round((1 / v - 1) * 2.0 ** 23)
    return (F32(1) / (F32(1) + (k * 2.0 ** -23).astype(F32))).astype(F32)


def score_ladder(n, hi=0.9995, lo=0.975):
    """n distinct float32 sigmoid values, descending"""
    s = sc(np.linspace(hi, lo, max(n, 1))[:n])
    assert len(np.unique(s)) == n
    return s


# ---------------------------------------------------------------------------------------------------------------------------------------
# box layouts (pixels, 0.5 grid)
# ---------------------------------------------------------------------------------------------------------------------------------------
def half(v):
    return (np.round(np.asarray(v, np.float64) * 2) / 2).astype(F32)


def cluster_boxes(n, rng, x0=0.0, y0=0.0):
    """random boxes, dense enough that NMS suppresses a good share of them"""
    side = max(40.0, 14.0 * np.sqrt(n))
    x1, y1 = half(x0 + rng.uniform(0, side, n)), half(y0 + rng.uniform(0, side, n))
    w, h = half(rng.uniform(4, 40, n)), half(rng.uniform(4, 40, n))
    return np.stack([x1, y1, x1 + w, y1 + h], 1).astype(F32)


def grid_boxes(n, x0=0.0, y0=0.0, cols=256):
    """disjoint 8 x 8 boxes at a 12-pixel pitch"""
    i = np.arange(n)
    x1, y1 = x0 + 12.0 * (i % cols), y0 + 12.0 * (i // cols)
    return np.stack([x1, y1, x1 + 8, y1 + 8], 1).astype(F32)


def chain_boxes(m, x0, y0):
    """a staircase: 20 x 10 boxes stepped by 6 pixels, IoU 14/26 with a neighbour, 8/32 with the next one, 0 further on"""
    x1 = x0 + 6.0 * np.arange(m)
    return np.stack([x1, np.full(m, y0), x1 + 20, np.full(m, y0 + 10.0)], 1).astype(F32)


def tv_iou(a, b):
    """torchvision's CPU nms IoU of two boxes, in its operation order, in float32"""
    a, b = torch.tensor(a, dtype=torch.float32), torch.tensor(b, dtype=torch.float32)
    ai, aj = (a[2] - a[0]) * (a[3] - a[1]), (b[2] - b[0]) * (b[3] - b[1])
    w = torch.clamp(torch.minimum(a[2], b[2]) - torch.maximum(a[0], b[0]), min=0)
    h = torch.clamp(torch.minimum(a[3], b[3]) - torch.maximum(a[1], b[1]), min=0)
    inter = w * h
    return (inter / (ai + aj - inter)).item()


def iou_pair(target):
    """two nested boxes sharing a corner, A = (a x b) / 2 px and B = (c x d) / 2 px with c <= a, d <= b, whose IoU in torchvision's
    float32 operation order (inter / (area_A + area_B - inter), inter = area_B) is exactly `target`; areas below 2^24 quarter pixels
    are exact, their sum is rounded like torchvision rounds it"""
    for a in range(4095, 3000, -1):
        for b in range(min(a, 16777215 // a), 3000, -1):
            u = F32(a * b)
            for p in (int(round(float(target) * a * b)) + dp for dp in (0, -1, 1)):
                pf = F32(p)
                if pf / ((u + pf) - pf) != target:
                    continue
                c = np.arange(max(1, -(-p // b)), a + 1)
                c = c[p % c == 0]
                if len(c):
                    return (0.0, 0.0, a / 2, b / 2), (0.0, 0.0, int(c[0]) / 2, p // int(c[0]) / 2)
    raise AssertionError(f"no box pair with IoU {target!r}")


def iou_targets(thr):
    f = F32(thr)
    return [np.nextafter(f, F32(0)), f, np.nextafter(f, F32(1))]


# ---------------------------------------------------------------------------------------------------------------------------------------
# 3-D anchor head cases (engine.DecodeNms.run)
# ---------------------------------------------------------------------------------------------------------------------------------------
def anchor_case(images, img_wh=(8192.0, 8192.0), seed=0, n_extra=48):
    """images: one dict per image with `boxes` [n, 4] and `scores` [n] (non-increasing) in the intended sorted order; optional
    `labels` [n] and `class_tie` [n] (every class gets the same logit: the first class wins).  Anchors: every image's candidates, then
    `n_extra` that never become candidates (score 0.5 below the threshold, masked out, or a prior with z mean <= 0), in a random index
    order; inside a run of equal scores the anchor indices ascend, so the intended order is the key (score desc, anchor index asc)."""
    rng = np.random.default_rng(seed)
    B = len(images)
    ns = [len(im["scores"]) for im in images]
    N = sum(ns) + n_extra
    perm = rng.permutation(N)
    cls = torch.zeros(B, N, NCLS_3D + 1)                       # logit 0: score 0.5, below the threshold
    cls[..., NCLS_3D] = torch.from_numpy(rng.choice(np.array([-1.0, 0.0, 1.0], F32), (B, N)))   # alpha_score 0.27 / exactly 0.5 / 0.73
    anchors = np.zeros((N, 4), F32)
    mask = torch.ones(B, N, dtype=torch.uint8)
    ms = np.zeros((N, T_3D, 6, 2), F32)
    ms[..., 0, 0] = half(rng.uniform(5, 60, (N, T_3D)))
    ms[..., 1, 0], ms[..., 2, 0] = rng.uniform(-1, 1, (N, T_3D)), rng.uniform(-1, 1, (N, T_3D))
    ms[..., 3:, 0] = half(rng.uniform(1, 4, (N, T_3D, 3)))
    ms[..., :, 1] = 1.0
    pos, labels_all, start = [], [], 0
    for b, im in enumerate(images):
        n = ns[b]
        idx = perm[start:start + n].copy()
        s = np.asarray(im["scores"], F32)
        assert bool((s[:-1] >= s[1:]).all())
        for v in np.unique(s):                                 # ascending anchor index inside each tie
            sel = np.nonzero(s == v)[0]
            idx[sel] = np.sort(idx[sel])
        anchors[idx] = im["boxes"]
        lab = np.asarray(im.get("labels", rng.integers(0, NCLS_3D, n)))
        tie = np.asarray(im.get("class_tie", np.zeros(n, bool)))
        lg = torch.from_numpy(logits_for(s))
        cls[b, idx, lab] = lg
        cls[b, idx[tie], :NCLS_3D] = lg[tie].unsqueeze(1)
        lab = np.where(tie, 0, lab)
        pos.append(idx)
        labels_all.append(lab)
        start += n
    extra = perm[start:]
    anchors[extra] = cluster_boxes(len(extra), rng, 0, 0)
    third = len(extra) // 3
    hi = torch.from_numpy(logits_for(np.full(len(extra), sc(0.99))))
    cls[:, extra[third:], 0] = hi[third:]                     # scores above the threshold ...
    mask[:, extra[third:2 * third]] = 0                        # ... but masked out
    ms[extra[2 * third:], :, 0, 0] = -1.0                      # ... or without a valid prior
    return dict(cls=cls.contiguous(), reg=torch.zeros(B, N, 12), anchors=torch.from_numpy(anchors), mean_std=torch.from_numpy(ms),
                mask=mask, img_w=float(img_wh[0]), img_h=float(img_wh[1]), pos=pos, labels=labels_all, n=ns)


def oracle_3d(case, b, thr):
    st = {}
    out = tp.get_bboxes(case["cls"][b], case["reg"][b], case["anchors"], case["mean_std"], case["mask"][b].bool(),
                        (case["img_h"], case["img_w"]), NCLS_3D, SCORE_THR_3D, thr, st)
    return out, st


def plain_image(n, seed, **kw):
    rng = np.random.default_rng(seed)
    tie = rng.random(n) < 0.25
    return dict(boxes=cluster_boxes(n, rng), scores=score_ladder(n), class_tie=tie, **kw)


COUNTS = [0, 1, 63, 64, 65, 1023, 1024, 1025, 2047, 2048]
CHAIN_BOUNDS = [64, 128, 1024, 2048]


def chain_image(n, first):
    """n disjoint boxes, except staircase chains over sorted positions first(B) .. first(B) + 5 for every B in CHAIN_BOUNDS"""
    boxes = grid_boxes(n, 0, 0)
    chains = []
    for i, B in enumerate(CHAIN_BOUNDS):
        p0 = first(B)
        boxes[p0:p0 + 6] = chain_boxes(6, 0, 4000 + 40 * i)
        chains.append(list(range(p0, p0 + 6)))
    return dict(boxes=boxes, scores=score_ladder(n)), chains


def tie_image(seed=0):
    """37 distinct scores, 300 equal ones (a staircase in anchor-index order across sorted positions 37 .. 336), 363 distinct below"""
    rng = np.random.default_rng(seed)
    top, low = score_ladder(37, lo=0.99), score_ladder(363, hi=0.98)
    tv = np.full(300, sc(0.985))
    assert top[-1] > tv[0] > low[0]
    boxes = np.concatenate([cluster_boxes(37, rng), chain_boxes(300, 0, 3000), cluster_boxes(363, rng)])
    return dict(boxes=boxes, scores=np.concatenate([top, tv, low]))


def iou_image(thr):
    """pairs (A, B) at sorted positions (2i, 2i + 1) whose IoU is float32(thr) and one ulp either side, plus disjoint fillers"""
    boxes, want = [], []
    for i, t in enumerate(iou_targets(thr)):
        a, b = iou_pair(t)
        off = np.array([3000.0 * i, 3000.0, 3000.0 * i, 3000.0], F32)
        boxes += [np.array(a, F32) + off, np.array(b, F32) + off]
        want.append(float(t) > thr)                            # B suppressed: the float32 IoU against the double threshold
    boxes = np.concatenate([np.stack(boxes), grid_boxes(40, 0, 0)])
    return dict(boxes=boxes, scores=score_ladder(len(boxes))), want


def degenerate_image(W=200.0, H=100.0):
    """boxes clipped to zero or negative width (0 / 0 and 0 / negative IoUs) among ordinary ones, image W x H"""
    raw = [[W + 4, 10, W + 12, 20], [W + 4, 10, W + 12, 20],      # past the right edge: x1 > x2 = W after clipping, twice
           [-12, 10, -4, 20], [-12, 30, -4, 40],                  # left of the image: x1 = 0 > x2
           [-8, 50, 0, 60], [-8, 50, 0, 60],                      # zero width: area 0, IoU 0 / 0 with its twin
           [W - 8, 10, W + 12, 20], [W - 8, 12, W + 20, 22],      # clipped at the right edge, overlapping
           [10, 10, 18, 20], [10, 10, 18, 20], [12, 10, 20, 20],  # ordinary ones
           [30, -6, 40, 4], [30, H - 4, 40, H + 6], [-4, -4, 4, 4]]
    raw = np.array(raw, F32)
    return dict(boxes=raw, scores=score_ladder(len(raw)))


# ---------------------------------------------------------------------------------------------------------------------------------------
# RetinaNet cases (RetinaDecode.run_levels) and the host restatement of the reference's decode
# ---------------------------------------------------------------------------------------------------------------------------------------
def retina_case(scores, boxes, level_pix, A, C, seed=0, class_tie=None):
    """scores [B, N] float32 (exact), boxes [N, 4]: the label of anchor n is a random class, given the score's logit; the other classes
    get logit -110 (score 0), or the same logit where `class_tie` is set.  Head outputs per level as the detector lays them out: NHWC
    [B, pix, cs] with channel pitches padded past A * C and A * 4, the padding filled with values that would win if it were read."""
    rng = np.random.default_rng(seed)
    scores = np.atleast_2d(np.asarray(scores, F32))
    B, N = scores.shape
    assert N == A * sum(level_pix)
    lab = rng.integers(0, C, (B, N))
    cls = torch.full((B, N, C), -110.0)
    lg = torch.from_numpy(logits_for(scores.reshape(-1)).reshape(B, N))
    cls.scatter_(2, torch.from_numpy(lab).unsqueeze(2), lg.unsqueeze(2))
    if class_tie is not None:
        cls[torch.from_numpy(np.asarray(class_tie))] = lg[torch.from_numpy(np.asarray(class_tie))].unsqueeze(1).expand(-1, C).clone()
    reg = torch.zeros(B, N, 4)
    cls_cs, reg_cs = (A * C + 15) // 16 * 16 + 16, A * 4 + 4
    cls_lv, reg_lv, o = [], [], 0
    for p in level_pix:
        c = torch.full((B, p, cls_cs), 30.0)
        c[..., :A * C] = cls[:, o:o + p * A].reshape(B, p, A * C)
        r = torch.full((B, p, reg_cs), 7.0)
        r[..., :A * 4] = reg[:, o:o + p * A].reshape(B, p, A * 4)
        cls_lv.append(c)
        reg_lv.append(r)
        o += p * A
    return dict(cls=cls, reg=reg, anchors=torch.from_numpy(np.asarray(boxes, F32)), cls_lv=cls_lv, reg_lv=reg_lv, level_pix=list(level_pix),
                cls_cs=cls_cs, reg_cs=reg_cs, A=A, C=C, N=N, B=B)


def retina_select(max_score, nms_pre):
    """the documented selection rule: the k = min(nms_pre, N) best by (score desc, anchor index asc)"""
    N = len(max_score)
    k = nms_pre if 0 < nms_pre < N else N
    order = torch.sort(max_score, descending=True, stable=True).indices
    return order[:k]


def retina_restate(cls, reg, anchors, nms_pre, means, stds, score_thr, iou_thr):
    """RetinanetHead.get_bboxes (R/heads/retinanet_head.py:257-307) for one image with the selection rule above; the decode in the
    reference's expression order (:227-255); returns scores, boxes, labels, anchor indices"""
    from torchvision.ops import nms
    max_score, label = cls.sigmoid().max(dim=-1)
    sel = retina_select(max_score, nms_pre)
    a, p = anchors[sel], reg[sel]
    d = p * torch.tensor(stds, dtype=torch.float32).unsqueeze(0) + torch.tensor(means, dtype=torch.float32).unsqueeze(0)
    dx, dy, dw, dh = d[:, 0], d[:, 1], d[:, 2], d[:, 3]
    px, py = (a[:, 0] + a[:, 2]) * 0.5, (a[:, 1] + a[:, 3]) * 0.5
    pw, ph = a[:, 2] - a[:, 0], a[:, 3] - a[:, 1]
    gw, gh = pw * dw.exp(), ph * dh.exp()
    gx, gy = px + pw * dx, py + ph * dy
    boxes = torch.stack([gx - gw * 0.5, gy - gh * 0.5, gx + gw * 0.5, gy + gh * 0.5], dim=-1)
    s = max_score[sel]
    keep = nms(boxes, s, iou_thr)
    keep = keep[s[keep] > score_thr]
    return s[keep], boxes[keep], label[sel][keep], sel[keep]


def kth_untied(max_score, nms_pre):
    N = len(max_score)
    if not (0 < nms_pre < N):
        return True
    v = torch.sort(max_score, descending=True).values
    return bool(v[nms_pre - 1] != v[nms_pre])


def _adjacent_scores(n_run, k0=84010):
    """n_run consecutive float32 sigmoid values (1 / (1 + k 2^-23), k = k0 ..), descending, about two ulps apart; their keys ~bits
    cross one boundary of the lowest byte mid-run"""
    k = np.arange(k0, k0 + n_run, dtype=np.float64)
    return (F32(1) / (F32(1) + (k * 2.0 ** -23).astype(F32))).astype(F32)


def retina_cases():
    """name -> (case, nms_pre, score_thr, iou_thr)"""
    rng = np.random.default_rng(7)
    out = {}

    def add(name, scores, level_pix, A, C, nms_pre, score_thr=0.98, iou_thr=0.4, **kw):
        s = np.atleast_2d(scores)
        N = s.shape[1]
        out[name] = (retina_case(s, cluster_boxes(N, rng), level_pix, A, C, seed=len(out), **kw), nms_pre, score_thr, iou_thr)

    def shuffled(s):
        return rng.permutation(np.asarray(s, F32))

    add("N1000", shuffled(score_ladder(1000)), [120, 80], 5, 3, 1000)
    add("N1025", shuffled(score_ladder(1025)), [205], 5, 3, 1000)
    add("N5000", shuffled(score_ladder(5000)), [600, 300, 100], 5, 3, 1000)
    add("ragged5", np.stack([shuffled(score_ladder(855)), shuffled(score_ladder(855, hi=0.999))]), [61, 23, 7, 3, 1], 9, 3, 600)
    tied = np.concatenate([score_ladder(700, lo=0.986), np.full(2000, sc(0.985)), score_ladder(2300, hi=0.984)])
    add("tie2000_at_k", shuffled(tied), [1000], 5, 3, 1000)
    add("all_equal", np.full(3000, sc(0.99)), [600], 5, 3, 1000)
    add("k_ge_N_pre0", shuffled(score_ladder(1800)), [360], 5, 3, 0)
    add("k_ge_N_pre5000", shuffled(score_ladder(1800)), [360], 5, 3, 5000)
    sat = np.concatenate([np.ones(300, F32), score_ladder(400), np.zeros(800, F32)])
    add("saturated_k_in_zeros", shuffled(sat), [300], 5, 3, 1000)
    sat2 = np.concatenate([np.ones(1200, F32), score_ladder(300)])
    add("saturated_k_in_ones", shuffled(sat2), [300], 5, 3, 1000)
    adj = _adjacent_scores(40)
    low = np.concatenate([score_ladder(500, hi=0.9995, lo=0.9905), np.repeat(adj, 3), score_ladder(1000, hi=0.985, lo=0.975)])
    add("low_byte_at_k", shuffled(low), [324], 5, 3, 561)
    thr_s = score_ladder(1000)
    at_thr = np.concatenate([thr_s[:50], np.full(6, thr_s[50]), thr_s[51:]])
    add("score_eq_thr", shuffled(at_thr), [201], 5, 3, 800, score_thr=float(thr_s[50]))
    ct = rng.random((1, 1500)) < 0.3
    add("class_ties", shuffled(score_ladder(1500)), [300], 5, 3, 1000, class_tie=ct)
    return out


# ---------------------------------------------------------------------------------------------------------------------------------------
# CenterNet cases (MonoFlex / KM3D decode) and the documented peak rule
# ---------------------------------------------------------------------------------------------------------------------------------------
CN_HEADS = {"MonoFlex": {"hm": CN_NCLS, "bbox2d": 4, "hps": 20, "rot": 8, "dim": 3, "reg": 2, "depth": 1, "depth_uncertainty": 1,
                         "corner_uncertainty": 3},
            "KM3D": {"hm": CN_NCLS, "wh": 2, "hps": 18, "rot": 8, "dim": 3, "prob": 1, "reg": 2, "hm_hp": 9, "hp_offset": 2}}


def cn_maps(kind, peaks, seed=0, hm_fill=None):
    """head maps {name: [B, n, H, W]}: heat logit -10 (sigmoid far below 0.1) except at `peaks` (one list of (c, y, x, logit) per
    image, or (c, y, x, logit, box): the box regression at (y, x) decodes to box = (x1, y1, x2, y2), integers in image pixels); box
    regressions on the 0.5 grid so that box columns 0..3 are exact; the rest random."""
    rng = np.random.default_rng(seed)
    B = len(peaks)
    m = {}
    for n, ch in CN_HEADS[kind].items():
        m[n] = torch.from_numpy(rng.standard_normal((B, ch, CN_H, CN_W)).astype(F32))
    m["hm"].fill_(-10.0)
    for b, pk in enumerate(peaks):
        if hm_fill is not None and hm_fill[b] is not None:
            m["hm"][b].fill_(hm_fill[b])
        for c, y, x, lg, *_ in pk:
            m["hm"][b, c, y, x] = float(lg)
    m["dim"] = torch.from_numpy(rng.uniform(1, 4, (B, 3, CN_H, CN_W)).astype(F32))
    if kind == "MonoFlex":
        m["bbox2d"] = torch.from_numpy(half(rng.uniform(0.5, 3, (B, 4, CN_H, CN_W))))
    else:
        m["wh"] = torch.from_numpy(half(rng.uniform(1, 6, (B, 2, CN_H, CN_W))))
        m["reg"] = torch.from_numpy(half(rng.uniform(0, 1, (B, 2, CN_H, CN_W))))
        m["hm_hp"].fill_(-10.0)
        m["hp_offset"].zero_()
    for b, pk in enumerate(peaks):
        for c, y, x, _, *box in pk:
            if not box:
                continue
            x1, y1, x2, y2 = box[0]                            # quarters / eighths of integers: every step below is exact
            if kind == "MonoFlex":                             # 4 * (x - l, y - t, x + r, y + b)
                m["bbox2d"][b, :, y, x] = torch.tensor([x - x1 / 4, y - y1 / 4, x2 / 4 - x, y2 / 4 - y])
            else:                                              # 4 * (x + dx -+ w / 2, y + dy -+ h / 2)
                m["reg"][b, :, y, x] = torch.tensor([(x1 + x2) / 8 - x, (y1 + y2) / 8 - y])
                m["wh"][b, :, y, x] = torch.tensor([(x2 - x1) / 4, (y2 - y1) / 4])
    return m


def cn_P2(B):
    P = torch.tensor([[700.0, 0.0, 80.0, 45.0], [0.0, 700.0, 48.0, -0.3], [0.0, 0.0, 1.0, 0.005]])
    return P.unsqueeze(0).repeat(B, 1, 1).contiguous()


def cn_restate(kind, maps, b, score_thr, iou_thr, K=CN_K):
    """the decode's documented rule: peaks (3x3 max-pool equality, as the reference) above score_thr, ordered by (score desc, flat index
    (c, y, x) asc), the best K, box columns 0..3 in the reference's expressions, torchvision NMS; returns scores, flat indices, boxes 0..3"""
    from torchvision.ops import nms
    heat = torch.sigmoid(maps["hm"][b:b + 1])
    peak = (F.max_pool2d(heat, 3, stride=1, padding=1) == heat) & (heat > score_thr)
    hv = heat.reshape(-1)
    flat = torch.nonzero(peak.reshape(-1))[:, 0]
    order = torch.sort(hv[flat], descending=True, stable=True).indices
    flat = flat[order][:K]
    s = hv[flat]
    HW = CN_H * CN_W
    y, x = ((flat % HW) // CN_W).float(), (flat % CN_W).float()
    at = lambda name, ch: maps[name][b, ch].reshape(-1)[flat % HW]
    if kind == "MonoFlex":
        bx = torch.stack([x - at("bbox2d", 0), y - at("bbox2d", 1), x + at("bbox2d", 2), y + at("bbox2d", 3)], 1)
    else:
        xs, ys = x + at("reg", 0), y + at("reg", 1)
        bx = torch.stack([xs - at("wh", 0) / 2, ys - at("wh", 1) / 2, xs + at("wh", 0) / 2, ys + at("wh", 1) / 2], 1)
    bx = bx * 4
    bx[:, 0] = torch.clamp(bx[:, 0], min=0)
    bx[:, 1] = torch.clamp(bx[:, 1], min=0)
    bx[:, 2] = torch.clamp(bx[:, 2], max=4.0 * CN_W)
    bx[:, 3] = torch.clamp(bx[:, 3], max=4.0 * CN_H)
    keep = nms(bx, s, iou_thr)
    return s[keep], flat[keep], bx[keep]


def cn_oracle(kind, maps, b, score_thr, iou_thr):
    ob = {k: v[b:b + 1] for k, v in maps.items()}
    f = tp.km3d_get_bboxes if kind == "KM3D" else tp.monoflex_get_bboxes
    return f(ob, cn_P2(len(next(iter(maps.values()))))[b:b + 1], (4 * CN_H, 4 * CN_W), score_thr, iou_thr, K=CN_K)


def _isolated(n, scores, rng, classes=CN_NCLS):
    """n peaks on a lattice of stride 2 (no two adjacent), random classes"""
    cells = [(c, y, x) for c in range(classes) for y in range(1, CN_H - 1, 2) for x in range(1, CN_W - 1, 2)]
    pick = rng.choice(len(cells), n, replace=False)
    lg = logits_for(scores)
    return [cells[i] + (lg[j],) for j, i in enumerate(pick)]


SWEEP_N, SWEEP_PAIR, SWEEP_CHAIN = 90, 10, 61


def _sweep_peaks(rng):
    """SWEEP_N isolated peaks in score order with chosen boxes: disjoint 8 x 8 tiles, except a pair at sorted positions SWEEP_PAIR and
    SWEEP_PAIR + 1 nested at IoU exactly 0.5 (8 x 8 and 8 x 4 sharing a corner), and a staircase over positions SWEEP_CHAIN .. + 5
    (IoU 14/26 with a neighbour, 8/32 with the next one) that crosses sorted positions 63 / 64"""
    pk = _isolated(SWEEP_N, score_ladder(SWEEP_N), rng, classes=1)      # one class: the box regression maps are shared by all
    pk = [(int(k), y, x, lg) for (_, y, x, lg), k in zip(pk, rng.integers(0, CN_NCLS, SWEEP_N))]
    tiles = iter((10 * (i % 16) + 1, 10 * (i // 16) + 1) for i in range(96))
    boxes = []
    for p in range(SWEEP_N):
        if p in (SWEEP_PAIR, SWEEP_PAIR + 1):
            boxes.append((60, 70, 68, 78 if p == SWEEP_PAIR else 74))
        elif SWEEP_CHAIN <= p < SWEEP_CHAIN + 6:
            x1 = 1 + 6 * (p - SWEEP_CHAIN)
            boxes.append((x1, 70, x1 + 20, 80))
        else:
            x1, y1 = next(tiles)
            boxes.append((x1, y1, x1 + 8, y1 + 8))
    return [q + (bx,) for q, bx in zip(pk, boxes)]


def cn_cases():
    """name -> (peaks per image, hm_fill per image or None, tie_free: the reference's topk order is defined, plateau cells to check)"""
    rng = np.random.default_rng(3)
    s = score_ladder(200)
    lg = logits_for(s)
    cases = {}
    # plateaus: 2x2 and 3x3 of equal heat, saturated ones (different logits, all sigmoid 1.0), one next to a higher cell
    pl = []
    pl += [(0, 5 + dy, 5 + dx, lg[40]) for dy in range(2) for dx in range(2)]
    pl += [(1, 10 + dy, 20 + dx, lg[41]) for dy in range(3) for dx in range(3)]
    pl += [(2, 15 + dy, 30 + dx, v) for (dy, dx), v in zip([(0, 0), (0, 1), (1, 0), (1, 1)], (20.0, 22.0, 25.0, 30.0))]
    pl += [(0, 3 + dy, 30 + dx, 18.0) for dy in range(3) for dx in range(3)]
    pl += [(1, 17 + dy, 8 + dx, lg[60]) for dy in range(3) for dx in range(3)] + [(1, 16, 7, lg[10])]
    pl += [(2, 5 + dy, 5 + dx, lg[40]) for dy in range(2) for dx in range(2)]                 # the same plateau in another class
    pl += [(c, y, x, lg[100 + i]) for i, (c, y, x) in enumerate([(0, 21, 2), (2, 21, 14), (1, 1, 14), (0, 12, 12), (2, 9, 37)])]
    plateau_peaks = [(1, 17 + dy, 8 + dx) for dy in range(3) for dx in range(3) if (dy, dx) != (0, 0)]
    cases["plateaus"] = ([pl], None, False, dict(peaks=plateau_peaks, not_peaks=[(1, 17, 8)]))
    # every border and corner, and a 2x2 plateau in a corner
    H, W = CN_H, CN_W
    bd = [(0, 0, 0), (1, 0, W - 1), (2, H - 1, 0), (0, H - 1, W - 1), (1, 0, 17), (2, H - 1, 23), (0, 11, 0), (1, 13, W - 1)]
    bp = [(c, y, x, lg[i * 3]) for i, (c, y, x) in enumerate(bd)]
    bp += [(2, dy, W - 2 + dx, lg[50]) for dy in range(2) for dx in range(2)]
    cases["borders"] = ([bp], None, False, dict(peaks=[(c, y, x) for c, y, x in bd], not_peaks=[]))
    bp_only = [(c, y, x, lg[i * 3]) for i, (c, y, x) in enumerate(bd)]
    cases["borders_tie_free"] = ([bp_only], None, True, dict(peaks=[(c, y, x) for c, y, x in bd], not_peaks=[]))
    # exactly K and K + 1 peaks above the threshold (batch of two)
    cases["K_and_K+1"] = ([_isolated(CN_K, score_ladder(CN_K), rng), _isolated(CN_K + 1, score_ladder(CN_K + 1), rng)], None, True,
                          dict(peaks=[], not_peaks=[]))
    # class ties straddling K: 95 distinct peaks above 12 equal ones spread over the classes (5 of the 12 make the cut)
    tie = [(c, y, x, logits_for([sc(0.975)])[0]) for c in range(CN_NCLS) for (y, x) in [(0, 2), (6, 38), (22, 9), (14, 25)]]
    cases["class_ties_at_K"] = ([_isolated(95, score_ladder(95, hi=0.9995, lo=0.98), rng) + tie], None, False, dict(peaks=[], not_peaks=[]))
    # peak-capacity overflow: image 0 is one plateau of heat 0.5 over every cell of every class
    cases["overflow"] = ([[], pl], [0.0, None], False, dict(peaks=[], not_peaks=[]))
    # more than 64 kept rows, a suppression chain across sorted positions 63 / 64 and a pair at IoU exactly nms_iou_thr (kept)
    cases["sweep_words"] = ([_sweep_peaks(rng)], None, True, dict(peaks=[], not_peaks=[]))
    return cases


# ---------------------------------------------------------------------------------------------------------------------------------------
# CPU checks of the builders
# ---------------------------------------------------------------------------------------------------------------------------------------
def test_logits_reproduce_the_chosen_scores():
    s = np.concatenate([score_ladder(3000), _adjacent_scores(40), [F32(1), F32(0), sc(0.985)]])
    lg = logits_for(s)
    assert np.array_equal(torch.sigmoid(torch.from_numpy(lg)).numpy(), s)
    assert np.array_equal(sigmoid_f32(lg), s)
    assert torch.sigmoid(torch.tensor([17.0, -104.0])).tolist() == [1.0, 0.0]
    adj = _adjacent_scores(40).view(np.int32)
    assert bool((np.diff(adj) < 0).all()) and bool((np.diff(adj) >= -3).all())
    key = ~adj.astype(np.int64) & 0xFFFFFFFF
    assert len(np.unique(key >> 8)) == 2, "the run crosses one boundary of the lowest key byte"


def _sorted_anchor_order(st):
    s, idx = st["cand_scores"], st["cand_anchor_idx"]
    return idx[torch.sort(s, descending=True, stable=True).indices]


@pytest.mark.parametrize("n", COUNTS)
def test_anchor_counts_and_order(n):
    case = anchor_case([plain_image(n, seed=n)], seed=n)
    (rs, rb, rc, ridx), st = oracle_3d(case, 0, 0.4)
    assert len(st["cand_scores"]) == n
    assert torch.equal(_sorted_anchor_order(st), torch.from_numpy(case["pos"][0]).long())
    assert torch.equal(rb[:, :4], case["anchors"][ridx.long()]) if n else len(rs) == 0
    if n > 10:
        assert 0 < len(rs) < n, "NMS suppresses some, not all"


def test_anchor_labels_alpha_and_extras():
    case = anchor_case([plain_image(300, seed=1)], seed=1)
    (rs, rb, rc, ridx), st = oracle_3d(case, 0, 0.4)
    pos, lab = case["pos"][0], case["labels"][0]
    want = dict(zip(pos.tolist(), lab.tolist()))
    assert [want[int(i)] for i in st["cand_anchor_idx"]] == st["cand_labels"].tolist()
    assert bool((case["cls"][0, pos][:, 0] == case["cls"][0, pos][:, 1]).any()), "some class ties"
    a = case["cls"][0, ridx.long(), NCLS_3D]
    assert bool((a == 0).any()) and bool((a < 0).any())                     # alpha_score exactly 0.5 and below it
    base = torch.atan2(case["mean_std"][ridx.long(), rc, 1, 0], case["mean_std"][ridx.long(), rc, 2, 0]) / 2
    np.testing.assert_allclose(rb[:, 10].numpy(), (base + np.pi * (a < 0).float()).numpy(), atol=1e-6)


def test_anchor_chains_keep_alternate_links():
    for first in (lambda B: B - 3, lambda B: B - 2):
        im, chains = chain_image(2100, first)
        case = anchor_case([im], seed=5)
        (rs, rb, rc, ridx), st = oracle_3d(case, 0, 0.4)
        sup = {p for ch in chains for p in ch[1::2]}
        want = [int(case["pos"][0][p]) for p in range(2100) if p not in sup]
        assert ridx.tolist() == want
        for B in CHAIN_BOUNDS:      # the link across the 64-row block (and, at 2048, mask word) boundary: kept -> suppressed, or the reverse
            assert ((B in sup) and (B - 1 not in sup)) if first(B) == B - 3 else ((B - 1 in sup) and (B not in sup))


def test_anchor_ties_decide_by_index():
    im = tie_image()
    case = anchor_case([im], seed=2)
    (rs, rb, rc, ridx), st = oracle_3d(case, 0, 0.4)
    order = _sorted_anchor_order(st)
    assert torch.equal(order, torch.from_numpy(case["pos"][0]).long())
    tied = case["pos"][0][37:337]
    kept = set(ridx.tolist()) & set(tied.tolist())
    assert kept == set(tied[0::2].tolist()), "the lower anchor index of each tied link is kept"


@pytest.mark.parametrize("thr", [0.4, 0.5])
def test_iou_pairs_on_both_sides_of_the_threshold(thr):
    im, want = iou_image(thr)
    for i, t in enumerate(iou_targets(thr)):
        assert F32(tv_iou(im["boxes"][2 * i], im["boxes"][2 * i + 1])) == t
    assert want == ([False, True, True] if thr == 0.4 else [False, False, True])
    case = anchor_case([im], seed=9)
    (rs, rb, rc, ridx), st = oracle_3d(case, 0, thr)
    kept = set(ridx.tolist())
    for i, w in enumerate(want):
        assert int(case["pos"][0][2 * i]) in kept
        assert (int(case["pos"][0][2 * i + 1]) not in kept) == w


def test_degenerate_boxes():
    case = anchor_case([degenerate_image()], img_wh=(200.0, 100.0), seed=4, n_extra=0)
    (rs, rb, rc, ridx), st = oracle_3d(case, 0, 0.4)
    cb = st["cand_boxes"]
    wdt = cb[:, 2] - cb[:, 0]
    assert bool((wdt < 0).any()) and bool((wdt == 0).any())
    assert len(rs) > 0


def test_retina_restatement_matches_the_reference_outputs():
    """the restatement (selection by (score desc, index asc), decode, NMS, threshold) on the reference's own head outputs: the same
    top-k set as `max_score.topk(nms_pre)` and the reference's kept rows"""
    from conftest import load_fixture
    fx = load_fixture("retinanet_96x320")
    anchors = torch.tensor(fx["anchors_full"])
    for b in range(int(fx["meta"][2])):
        cls, reg = torch.tensor(fx["cls_full"][b]), torch.tensor(fx["reg_full"][b])
        ms = cls.sigmoid().max(-1).values
        assert kth_untied(ms, 1000)
        assert set(retina_select(ms, 1000).tolist()) == set(ms.topk(1000).indices.tolist()) == set(fx[f"topk_{b}"].tolist())
        s, bx, lab, idx = retina_restate(cls, reg, anchors, 1000, [0.0] * 4, [1.0] * 4, 0.2, 0.4)
        np.testing.assert_array_equal(idx.numpy(), fx[f"topk_{b}"][fx[f"keep_{b}"]][:len(s)])
        np.testing.assert_array_equal(lab.numpy(), fx[f"cls_{b}"])
        np.testing.assert_array_max_ulp(s.numpy(), fx[f"scores_{b}"], maxulp=1)
        np.testing.assert_array_max_ulp(bx.numpy(), fx[f"bboxes_{b}"], maxulp=2)


def test_retina_cases_are_what_they_claim():
    cases = retina_cases()
    for name, (c, nms_pre, score_thr, iou_thr) in cases.items():
        for b in range(c["B"]):
            ms = c["cls"][b].sigmoid().max(-1).values
            s, bx, lab, idx = retina_restate(c["cls"][b], c["reg"][b], c["anchors"], nms_pre, [0.0] * 4, [1.0] * 4, score_thr, iou_thr)
            assert torch.equal(bx, c["anchors"][idx]), name                   # reg = 0: the decode returns the anchors bit for bit
            assert len(s) > 0 and bool((s > score_thr).all()), name
            if kth_untied(ms, nms_pre):                                         # the reference's own call selects the same set
                k = nms_pre if 0 < nms_pre < c["N"] else c["N"]
                assert set(retina_select(ms, nms_pre).tolist()) == set(ms.topk(k).indices.tolist()), name
    tied = lambda n: not kth_untied(cases[n][0]["cls"][0].sigmoid().max(-1).values, cases[n][1])
    assert tied("tie2000_at_k") and tied("all_equal") and tied("saturated_k_in_zeros") and tied("saturated_k_in_ones")
    assert not tied("N1025") and not tied("N5000") and not tied("ragged5")
    ms = cases["tie2000_at_k"][0]["cls"][0].sigmoid().max(-1).values
    assert int((ms == sc(0.985)).sum()) == 2000 and int((ms > sc(0.985)).sum()) == 700
    ms = cases["low_byte_at_k"][0]["cls"][0].sigmoid().max(-1).values
    v = torch.sort(ms, descending=True).values
    kb = (~v[559:562].numpy().view(np.int32)).view(np.uint32)
    assert len(set((kb >> 8).tolist())) == 1 and len(set(kb.tolist())) > 1, "the k-th key is decided by the lowest byte"
    c, nms_pre, thr, _ = cases["score_eq_thr"]
    assert int((c["cls"][0].sigmoid().max(-1).values == F32(thr)).sum()) == 6
    c = cases["saturated_k_in_zeros"][0]
    ms = c["cls"][0].sigmoid().max(-1).values
    assert int((ms == 1).sum()) == 300 and int((ms == 0).sum()) == 800


@pytest.mark.parametrize("kind", ["MonoFlex", "KM3D"])
def test_centernet_cases_are_what_they_claim(kind):
    thr, iou = 0.1, 0.5
    for name, (peaks, fill, tie_free, extra) in cn_cases().items():
        maps = cn_maps(kind, peaks, seed=1, hm_fill=fill)
        for b in range(len(peaks)):
            heat = torch.sigmoid(maps["hm"][b:b + 1])
            pk = (F.max_pool2d(heat, 3, stride=1, padding=1) == heat) & (heat > thr)
            if fill is not None and fill[b] is not None:
                assert int(pk.sum()) == CN_NCLS * CN_H * CN_W                    # every cell of a flat map is a peak
                continue
            for c, y, x in extra["peaks"]:
                assert bool(pk[0, c, y, x]), (name, c, y, x)
            for c, y, x in extra["not_peaks"]:
                assert not bool(pk[0, c, y, x]), (name, c, y, x)
            s, flat, bx = cn_restate(kind, maps, b, thr, iou)
            rs, rb, rc, rflat = cn_oracle(kind, maps, b, thr, iou)
            if tie_free:
                assert torch.equal(flat, rflat) and torch.equal(s, rs) and torch.equal(bx, rb[:, :4]), name
            else:
                assert sorted(s.tolist()) == sorted(rs.tolist()) or name == "plateaus", name
    peaks = cn_cases()["K_and_K+1"][0]
    assert [len(p) for p in peaks] == [CN_K, CN_K + 1]
    pk = cn_cases()["sweep_words"][0][0]
    s, flat, bx = cn_restate(kind, cn_maps(kind, [pk], seed=1), 0, thr, iou)
    kept = [p for p in range(SWEEP_N) if p not in (SWEEP_CHAIN + 1, SWEEP_CHAIN + 3, SWEEP_CHAIN + 5)]   # 63 kept suppresses 64
    assert SWEEP_CHAIN + 3 == 64 and len(kept) > 64
    assert flat.tolist() == [(pk[p][0] * CN_H + pk[p][1]) * CN_W + pk[p][2] for p in kept]
    assert torch.equal(bx, torch.tensor([pk[p][4] for p in kept], dtype=torch.float32))
    assert F32(tv_iou(pk[SWEEP_PAIR][4], pk[SWEEP_PAIR + 1][4])) == F32(iou)
    maps = cn_maps(kind, cn_cases()["plateaus"][0], seed=1)
    heat = torch.sigmoid(maps["hm"])
    assert int((heat[0, 2, 15:17, 30:32] == 1).sum()) == 4 and int((heat[0, 0, 3:6, 30:33] == 1).sum()) == 9
