"""One eager YOLOStereo3D step (batch 8, 384x1280, the bench's stereo config) under torch.profiler: every kernel in launch order with its
device time, then the busy time per kernel name.  Run it on its own (tracing slows the host).
usage: python tools/prof_step.py [--out DIR]"""
import argparse
import collections
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the kernel list to DIR/prof_step.txt")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "prof_step needs a GPU"
    from visualdet3d_b200 import synth
    from visualdet3d_b200.detectors import build_synthetic_stereo3d
    B, H, W = 8, 384, 1280
    det = build_synthetic_stereo3d(seed=0)[0].cuda().eval()
    left, right, P2, P3 = (t.cuda() for t in synth.synth_stereo_inputs(B, H, W, seed=1))
    with torch.no_grad():
        for _ in range(3):
            det.forward_batch(left, right, P2, P3)
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            det.forward_batch(left, right, P2, P3)
            torch.cuda.synchronize()
    ks = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and e.device_time > 0 and "Memcpy" not in e.name
                 and "Memset" not in e.name), key=lambda e: e.time_range.start)
    lines = [f"{i:4d} {e.device_time:9.1f} us  {e.name[:110]}" for i, e in enumerate(ks)]
    tot = collections.Counter()
    for e in ks:
        tot[e.name.split("<")[0].split("(")[0]] += e.device_time
    busy = sum(e.device_time for e in ks)
    lines.append(f"{len(ks)} kernels, {busy / 1e3:.2f} ms busy")
    lines += [f"  {v / 1e3:8.3f} ms  {100 * v / busy:5.1f} %  {k}" for k, v in tot.most_common(12)]
    print("\n".join(lines), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "prof_step.txt"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
