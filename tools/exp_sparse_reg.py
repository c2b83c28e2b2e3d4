"""The anchor head's regression output conv on the decoder's rows only.
  count: on the bench's own seeded inputs and shapes, the anchors that pass the anchor mask and the score threshold (the candidates
         decode_candidates_kernel decodes) and the (pixel, anchor group) pairs that hold at least one of them, against the dense reg_out
         conv's 128-pixel tiles
  time:  CUDA-event time of the dense reg_out conv against the candidate list + the gathered-row conv, with the list's entry count and the
         card's name, power limit and SM clock
usage: python tools/exp_sparse_reg.py count|time [reps]"""
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from visualdet3d_b200 import synth                                      # noqa: E402
from visualdet3d_b200.detectors import build_synthetic_mono3d, build_synthetic_stereo3d      # noqa: E402

CONFIGS = {"stereo": (384, 1280, 8), "gac": (288, 1280, 8), "yolo3d": (288, 1280, 1)}


def build(config):
    if config == "stereo":
        return build_synthetic_stereo3d(seed=0)[0]
    if config == "gac":
        return build_synthetic_mono3d("GroundAwareYolo3D", seed=0)[0]
    return build_synthetic_mono3d("Yolo3D", seed=0, depth=18)[0]


def inputs(config, B, H, W):
    if config == "stereo":
        l, r, p2, _ = synth.synth_stereo_inputs(B, H, W, seed=1)
        return [l.cuda(), r.cuda(), p2.cuda()]
    im, p2 = synth.synth_mono_inputs(B, H, W, seed=1)
    return [im.cuda(), p2.cuda()]


def count(config):
    H, W, B = CONFIGS[config]
    det = build(config).cuda().eval()
    seen = {}
    det.stage_hook = lambda name, v: seen.__setitem__(name, v.clone() if isinstance(v, torch.Tensor) else v.t.clone())
    with torch.no_grad():
        det.launch(*inputs(config, B, H, W))
    torch.cuda.synchronize()
    A, ncls = det.num_anchors, det.num_classes
    cls, mask = seen["cls_preds"], seen["mask"].bool()
    h, w = H // 16, W // 16
    best = torch.sigmoid(cls.view(B, h * w * A, -1)[..., :ncls]).max(-1).values
    cand = (mask & (best > det.test_cfg["score_thr"])).view(B, h * w, A)
    m_tiles = B * -(-h // 8) * -(-w // 16)
    print(f"{config}: B={B} {H}x{W} map {h}x{w} anchors/px {A}  candidates {int(cand.sum())} "
          f"({int(cand.sum()) / B:.0f} per image, {100.0 * float(cand.float().mean()):.2f} % of anchors), mask {100.0 * float(mask.float().mean()):.1f} %")
    print(f"  dense reg_out: {m_tiles} pixel tiles x {A * 12} columns")
    for g in (4, 8, 16):
        if A % g:
            continue
        pairs = cand.view(B, h * w, A // g, g).any(-1)
        per_group = pairs.sum((0, 1))
        tiles = int(sum(-(-int(c) // 128) for c in per_group))
        print(f"  group {g:2d} anchors ({12 * g} cols): {int(pairs.sum())} pairs ({int(pairs.sum()) / B:.0f} per image), "
              f"{tiles} tiles of 128 rows -> {tiles * 12 * g / (m_tiles * A * 12) * 100:.1f} % of the dense MMA work")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name()


def events(fn, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    return float(np.median(ts)), float(min(ts))


def time_config(config, reps):
    from visualdet3d_b200 import engine as E
    H, W, B = CONFIGS[config]
    det = build(config).cuda().eval()
    x = inputs(config, B, H, W)
    with torch.no_grad():
        os.environ["VD3D_SPARSE_REG"] = "1"
        det.launch(*x)                          # fills the arena: mask, REG (and on the sparse path the list and counts)
        pl = det.prepare()
        ro = pl["reg_out"]
        if config == "stereo":
            _, cls, r3 = det.core_forward(x[0], x[1], reg_out=False)
        else:
            feat = pl["backbone"].run(x[0], det._arena)[0]
            if pl["backbone"].last_lo_stale:
                E.split_lo(feat)
            cls = E.Act(det._arena.get("CLS", (B, H // 16, W // 16, pl["cls"][2].Cout), x[0].device))
            r3 = det.run_reg(pl, feat, x[-1], det._arena)
        ar = det._arena
        N = B * r3.H * r3.W * det.num_anchors
        mask = ar.get("mask", (B, N // B), x[0].device, dtype=torch.uint8)
        groups = -(-det.num_anchors // E.REG_GROUP_ANCHORS)
        lst = ar.get("reg_list", (groups, B * r3.H * r3.W), x[0].device, dtype=torch.int32)
        counts = ar.get("reg_counts", (groups,), x[0].device, dtype=torch.int32)
        sparse_path = det.sparse_reg(ro, B, r3.H, r3.W)
        reg = ar.act("REG", (B, r3.H, r3.W, ro.Cout), x[0].device)
        thr = det.test_cfg["score_thr"]

        def sparse():
            E.reg_candidates(cls.t, mask, det.num_anchors, det.num_classes, thr, lst, counts)
            ro.gather(r3, lst, counts, reg)

        for _ in range(3):
            ro(r3, reg), sparse()
        d, dmin = events(lambda: ro(r3, reg), reps)
        s, smin = events(sparse, reps)
        c = counts.cpu().tolist()
        tiles = sum(-(-n // 128) for n in c)
    print(f"{config}: B={B} {H}x{W} reg_out {r3.C} -> {ro.Cout}: dense {d:8.1f} us (min {dmin:.1f})   list + gathered {s:7.1f} us (min {smin:.1f})"
          f"   entries {sum(c)} in {groups} groups = {tiles} tiles of 128 rows   ({d / s:.2f}x; the detector takes the "
          f"{'gathered' if sparse_path else 'dense'} path)", flush=True)


if __name__ == "__main__":
    mode = sys.argv[1] if len(sys.argv) > 1 else "count"
    print(card(), flush=True)
    for c in ("stereo", "gac", "yolo3d"):
        if mode == "count":
            count(c)
        else:
            time_config(c, int(sys.argv[2]) if len(sys.argv) > 2 else 50)
    print(card(), flush=True)
