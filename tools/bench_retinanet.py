"""RetinaNet 2-D detector on the GPU (example config: ResNet-50, FPN P3..P7, 4 + 4 head convs of 256 channels), device-resident synthetic input.

    python tools/bench_retinanet.py [--H 288 --W 1280 --batches 1,8 --steps 30 --warmup 5 --reps 50]

Prints JSON lines: per batch size the images/s of the whole step (CUDA events, no host sync inside the window), kernel launches per step,
per-stage event times (backbone, FPN, head, decode) and the head's achieved TFLOP/s (FLOPs counted from the shapes below); then one 256 -> 256
head layer as one multi-level launch against the same layer launched level by level (CUDA-graph replays, alternating, in this process); the
card's name and power limit come from the same run.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402
from bench_common import card  # noqa: E402


def head_flops(det, hws, B):
    """multiply-adds x 2 of the head over all levels: 2 x stacked_convs 3x3 convs feat -> feat, the cls (A * C) and reg (A * 4) output convs"""
    hd = det.bbox_head
    per_pix = 0
    for tower in (hd.cls_conv, hd.reg_conv):
        for m in tower:
            c = m.sequence[0]
            per_pix += 2 * 9 * c.in_channels * c.out_channels
    for c in (hd.retina_cls[0], hd.retina_reg[0]):
        per_pix += 2 * 9 * c.in_channels * c.out_channels
    return per_pix * B * sum(h * w for h, w in hws)


def ev():
    e = torch.cuda.Event(enable_timing=True)
    e.record()
    return e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--H", type=int, default=288)
    ap.add_argument("--W", type=int, default=1280)
    ap.add_argument("--batches", default="1,8")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_retinanet: needs a CUDA device")
    from visualdet3d_b200 import _lib, synth
    from visualdet3d_b200.detectors import build_synthetic_retinanet
    det, _, _ = build_synthetic_retinanet(seed=0)
    det = det.cuda().eval()
    gpu = card()
    for B in [int(v) for v in a.batches.split(",")]:
        img, _ = synth.synth_mono_inputs(B, a.H, a.W, seed=1)
        img = img.cuda()
        with torch.no_grad():
            for _ in range(a.warmup):
                det.launch(img)
            torch.cuda.synchronize()
            n0 = _lib.launch_count()
            det.launch(img)
            torch.cuda.synchronize()
            launches = _lib.launch_count() - n0
            e0 = ev()
            for _ in range(a.steps):
                det.launch(img)
            e1 = ev()
            torch.cuda.synchronize()
            step_ms = e0.elapsed_time(e1) / a.steps
            # per-stage times: the same launches with events between the stages
            st = {k: 0.0 for k in ("backbone", "fpn", "head", "decode")}
            for _ in range(a.steps):
                t0 = ev(); feats = det.backbone(img)
                t1 = ev(); levels = det.fpn(feats)
                t2 = ev(); heads = det.head(levels)
                t3 = ev(); det.decode(heads, a.H, a.W)
                t4 = ev()
                torch.cuda.synchronize()
                for k, (x, y) in zip(st, ((t0, t1), (t1, t2), (t2, t3), (t3, t4))):
                    st[k] += x.elapsed_time(y) / a.steps
        hws = [(x.H, x.W) for x in levels]
        fl = head_flops(det, hws, B)
        print(json.dumps({"metric": "retinanet_images_per_sec", "H": a.H, "W": a.W, "batch": B, "value": B * 1000.0 / step_ms,
                          "ms_per_step": step_ms, "launches_per_step": launches, "stage_ms": st, "head_gflop": fl / 1e9,
                          "head_tflops": fl / (st["head"] * 1e-3) / 1e12, "card": gpu, "steps": a.steps,
                          "warmup": a.warmup}))
        # one head layer: one multi-level launch vs level-by-level launches of the same layer, alternating
        from visualdet3d_b200 import engine as E
        layer = det.prepare()["cls"][1]
        ar = E.Arena()
        xs = ar.level_acts("bench.x", B, hws, layer.Cin, "cuda", lo=True)
        for x in xs:
            x.t.normal_()
            E.split_lo(x)
        grouped_out = ar.level_acts("bench.g", B, hws, layer.Cout, "cuda", lo=True)
        per_out = [ar.act(f"bench.p{i}", (B, h, w, layer.Cout), "cuda", lo=True) for i, (h, w) in enumerate(hws)]
        # each form captured in a CUDA graph of K back-to-back calls and replayed alternately: the replays time the device work only (the
        # eager calls also encode the tensor maps on the host, which a batch-1 layer does not hide)
        K = 10

        def grouped():
            layer.run_levels(xs, grouped_out)

        def per_level():
            for x, o in zip(xs, per_out):
                layer(x, o)
        graphs = []
        with torch.no_grad():
            for fn in (grouped, per_level):
                fn()
                torch.cuda.synchronize()
                gr = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gr, capture_error_mode="thread_local"):
                    for _ in range(K):
                        fn()
                graphs.append(gr)
            tg = tp = 0.0
            for r in range(a.warmup + a.reps):
                g0 = ev(); graphs[0].replay(); g1 = ev(); graphs[1].replay(); p1 = ev()
                torch.cuda.synchronize()
                if r >= a.warmup:
                    tg += g0.elapsed_time(g1) / (a.reps * K)
                    tp += g1.elapsed_time(p1) / (a.reps * K)
        lf = 2 * 9 * layer.Cin * layer.Cout * B * sum(h * w for h, w in hws)
        print(json.dumps({"metric": "retinanet_head_layer_grouped_vs_per_level", "H": a.H, "W": a.W, "batch": B, "grouped_us": tg * 1e3,
                          "per_level_us": tp * 1e3, "grouped_tflops": lf / (tg * 1e-3) / 1e12, "per_level_tflops": lf / (tp * 1e-3) / 1e12,
                          "levels": hws, "card": gpu, "reps": a.reps}))


if __name__ == "__main__":
    main()
