"""The anchor head's regression tower on the tiles its candidates reach (Anchor3DDetector.decode's `tower`).
On the bench's own seeded inputs and shapes (stereo: batch 8, 384x1280; gac: batch 8, 288x1280), per tower conv:
  * the 8 x 16 tiles of its device list (vd3d_reg_tower_tiles) against the dense conv's tiles;
  * the CUDA-event time (median of `reps` launches) of the dense conv, the tile-listed conv on the detector's lists, and the tile-listed conv
    on full-map lists (every pixel a candidate: the worst case, the dense tile count plus the store-map reads);
  * the time of the list building itself: vd3d_reg_candidates with the pixel map + vd3d_reg_tower_tiles, against vd3d_reg_candidates alone.
Prints the card's name, power limit, SM clock and power draw before and after.
usage: python tools/exp_sparse_tower.py [reps]"""
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from visualdet3d_b200 import engine as E, synth                                            # noqa: E402
from visualdet3d_b200.detectors import build_synthetic_mono3d, build_synthetic_stereo3d     # noqa: E402

CONFIGS = {"stereo": (384, 1280, 8), "gac": (288, 1280, 8)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,power.draw", "--format=csv,noheader"],
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


def run(config, reps):
    H, W, B = CONFIGS[config]
    if config == "stereo":
        det = build_synthetic_stereo3d(seed=0)[0].cuda().eval()
        l, r, p2, _ = synth.synth_stereo_inputs(B, H, W, seed=1)
        x = [l.cuda(), r.cuda(), p2.cuda()]
    else:
        det = build_synthetic_mono3d("GroundAwareYolo3D", seed=0)[0].cuda().eval()
        im, p2 = synth.synth_mono_inputs(B, H, W, seed=1)
        x = [im.cuda(), p2.cuda()]
    ar, dev = det._arena, x[0].device
    with torch.no_grad():
        pl = det.prepare()
        tower = det.reg_tower(pl)
        assert det.tower_tiles_ok(tower, pl["reg_out"], H // 16, W // 16)
        det.launch(*x)                                   # the tiled path: fills the candidate map, the lists and the counts
        if config == "stereo":
            _, cls, feat = det.core_forward(x[0], x[1], reg_out=False, reg_tower=False)
        else:
            f = pl["backbone"].run(x[0], ar)[0]
            if pl["backbone"].last_lo_stale:
                E.split_lo(f)
            cls = E.Act(ar.get("CLS", (B, H // 16, W // 16, pl["cls"][2].Cout), dev))
            feat = det.run_reg(pl, f, x[-1], ar, tower=False)
        h, w, D = feat.H, feat.W, len(tower)
        cap = E.tower_tile_cap(B, h, w)
        pix = ar.get("reg_pix", (B, h, w), dev, dtype=torch.uint8)
        smaps = ar.get("tower_smap", (D, B, h, w), dev, dtype=torch.uint8)
        tiles = ar.get("tower_tiles", (D, cap, 4), dev, dtype=torch.int32)
        tcount = ar.get("tower_count", (D,), dev, dtype=torch.int32)
        counts = tcount.cpu().tolist()
        # full-map lists: every pixel a candidate
        f_smaps, f_tiles, f_count = torch.empty_like(smaps), torch.empty_like(tiles), torch.empty_like(tcount)
        E.tower_tiles(torch.ones_like(pix), f_smaps, f_tiles, f_count)
        # the dense chain once, so that every input below is valid everywhere
        ins, outs = [], []
        a = feat
        for layer, name, res in tower:
            o = ar.act(name, (B, h, w, layer.Cout), dev, lo=True)
            rr = outs[res] if res is not None else None
            ins.append((a, o, rr))
            a = layer(a, o, res=rr)
            outs.append(a)
        dense_tiles = B * -(-h // 8) * -(-w // 16)
        print(f"{config}: B={B} {H}x{W} map {h}x{w}, candidate pixels {int(pix.sum())} of {B * h * w}, dense {dense_tiles} tiles per conv",
              flush=True)
        tot = [0.0, 0.0, 0.0]
        for j, (layer, name, res) in enumerate(tower):
            d = D - j
            xi, o, rr = ins[j]
            lst = (tiles[d - 1], tcount[d - 1:d], smaps[d - 1])
            full = (f_tiles[d - 1], f_count[d - 1:d], f_smaps[d - 1])
            for fn in (lambda: layer(xi, o, res=rr), lambda: layer(xi, o, res=rr, tiles=lst), lambda: layer(xi, o, res=rr, tiles=full)):
                fn()
            t_d, _ = events(lambda: layer(xi, o, res=rr), reps)
            t_t, _ = events(lambda: layer(xi, o, res=rr, tiles=lst), reps)
            t_f, _ = events(lambda: layer(xi, o, res=rr, tiles=full), reps)
            tot[0] += t_d; tot[1] += t_t; tot[2] += t_f
            S = int(smaps[d - 1].sum())
            print(f"  {name} ({layer.Cin} -> {layer.Cout}, depth {d}): S_d {100.0 * S / (B * h * w):5.1f} % of the pixels, "
                  f"{counts[d - 1]:4d} / {dense_tiles} tiles   dense {t_d:8.1f} us   tiled {t_t:8.1f} us ({t_d / t_t:.2f}x)   "
                  f"full-map list {t_f:8.1f} us ({t_f - t_d:+.1f} us)", flush=True)
        print(f"  tower: dense {tot[0]:.1f} us, tiled {tot[1]:.1f} us (saves {tot[0] - tot[1]:.1f} us), full-map list {tot[2]:.1f} us "
              f"({tot[2] - tot[0]:+.1f} us)", flush=True)
        # list building
        A = det.num_anchors
        mask = ar.get("mask", (B, h * w * A), dev, dtype=torch.uint8)
        groups = -(-A // E.REG_GROUP_ANCHORS)
        lst = ar.get("reg_list", (groups, B * h * w), dev, dtype=torch.int32)
        cnt = ar.get("reg_counts", (groups,), dev, dtype=torch.int32)
        thr = det.test_cfg["score_thr"]
        cand = lambda: E.reg_candidates(cls.t, mask, A, det.num_classes, thr, lst, cnt)

        def build():
            E.reg_candidates(cls.t, mask, A, det.num_classes, thr, lst, cnt, pix)
            E.tower_tiles(pix, smaps, tiles, tcount)
        for _ in range(3):
            cand(), build()
        t_c, _ = events(cand, reps)
        t_b, _ = events(build, reps)
        print(f"  lists: candidates {t_c:.1f} us, candidates + pixel map + tower tiles {t_b:.1f} us ({t_b - t_c:+.1f} us)", flush=True)


if __name__ == "__main__":
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 50
    print(card(), flush=True)
    for c in CONFIGS:
        run(c, reps)
    print(card(), flush=True)
