"""Time Stereo3D's disparity loss, forward + backward, native (visualdet3d_b200/disparity_loss.py) against the reference's
`DisparityLoss(96)` on CUDA tensors, on the same GPU, at D = 96 and 72x320 maps (the Stereo3D_example training shape's 1/4 resolution):
B = 4 (the training batch) and B = 16 (a bandwidth reading at a larger volume).  The logits are randn * 2 and the label is
tests/golden/disparity_loss.npz case a's (regenerated from its seed; B = 16 repeats its 4 images 4 times).

Reports, per arm: ms per step (host clock around steps ending in a device synchronise, after warm-up); from one profiled step, kernel
launches, device-to-host copies and host synchronisations; the peak memory allocated over one step above what was allocated before it.
For the native kernels alone: the forward (both launches) and the backward timed by CUDA events over many back-to-back launches, with
their algorithmic bytes (forward B*D*H*W*4 + B*H*W*(4 + 4), backward 2*B*D*H*W*4 + B*H*W*(4 + 4)) as GB/s and as a share of 3.35 TB/s.
Prints the card's name, power limit and max SM clock; writes nothing.

    python tools/bench_disparity_loss.py [--steps 50] [--warmup 10] [--launches 200]
The reference arm needs the reference package (oracle/_ref/visualDet3D or the reference tree); without it only the native arm runs."""
import argparse
import importlib.util
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402
from bench_common import card, timed  # noqa: E402

HBM_BYTES_PER_S = 3.35e12        # H100 SXM5 80 GB HBM3


def peak_bytes(step):
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    step()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - before


def event_ms(fn, launches):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / launches


def kernels(x, label, launches):
    """The native forward (two launches) and backward alone, on preallocated buffers."""
    from visualdet3d_b200 import _lib
    lib = _lib.load()
    B, D, H, W = x.shape
    ws_bytes = int(lib.vd3d_disparity_loss_workspace_bytes(B, D, H, W))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    lse = torch.empty(B, H, W, device="cuda")
    loss = torch.empty((), device="cuda")
    g = torch.ones((), device="cuda")
    grad = torch.empty_like(x)
    st = torch.cuda.current_stream().cuda_stream
    fwd = lambda: lib.vd3d_disparity_loss_forward(x.data_ptr(), label.data_ptr(), B, D, H, W, ws.data_ptr(), ws_bytes,  # noqa: E731
                                                  lse.data_ptr(), loss.data_ptr(), st)
    bwd = lambda: lib.vd3d_disparity_loss_backward(x.data_ptr(), label.data_ptr(), lse.data_ptr(), B, D, H, W, g.data_ptr(),  # noqa: E731
                                                   grad.data_ptr(), st)
    out = {}
    vol, pix = B * D * H * W * 4, B * H * W * 4
    for name, fn, nbytes in (("forward", fwd, vol + 2 * pix), ("backward", bwd, 2 * vol + 2 * pix)):
        ms = event_ms(fn, launches)
        gbs = nbytes / (ms * 1e-3) / 1e9
        out[name] = dict(us=round(ms * 1e3, 2), algorithmic_bytes=nbytes, GB_per_s=round(gbs, 1),
                         share_of_3_35_TB_s=round(gbs * 1e9 / HBM_BYTES_PER_S, 3))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    import refload
    from visualdet3d_b200 import _lib, disparity_loss
    spec = importlib.util.spec_from_file_location("gen", os.path.join(ROOT, "tests", "golden", "make_golden_disparity_loss.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    _, label4 = gen.inputs("a")
    D, H, W = 96, int(label4.shape[1]), int(label4.shape[2])
    rec = dict(card=card(), torch=torch.__version__, steps=args.steps, warmup=args.warmup, launches=args.launches, D=D, H=H, W=W,
               valid_fraction=round(float(((label4 > 0) & (label4 < D)).float().mean()), 4))
    shapes = {}
    for B in (4, 16):
        g = torch.Generator().manual_seed(B)
        x = (torch.randn(B, D, H, W, generator=g) * 2).cuda().requires_grad_(True)
        label = torch.cat([label4] * (B // 4)).cuda()
        shapes[B] = (x, label)

        def native():
            x.grad = None
            disparity_loss.disparity_loss(x, label, D).backward()

        r = dict(volume_MB=round(x.numel() * 4 / 1e6, 1), native=timed(native, args.steps, args.warmup))
        _lib.launch_count_reset()
        native()
        torch.cuda.synchronize()
        r["native"]["native_launches"] = _lib.launch_count()
        r["native"]["peak_alloc_MB"] = round(peak_bytes(native) / 1e6, 2)
        r["native_kernels"] = kernels(x.detach(), label, args.launches)
        rec[f"B{B}"] = r
    if refload.available():
        from visualdet3d_b200.ops import dcn, iou3d
        refload.load_reference(device="cuda", dcn_ext=dcn, iou3d_ext=iou3d)
        from visualDet3D.networks.heads.losses import DisparityLoss
        ref = DisparityLoss(D)
        for B, (x, label) in shapes.items():
            def reference():
                x.grad = None
                ref(x, label).backward()

            r = rec[f"B{B}"]
            r["reference"] = timed(reference, args.steps, args.warmup)
            r["reference"]["peak_alloc_MB"] = round(peak_bytes(reference) / 1e6, 2)
            r["speedup"] = round(r["reference"]["ms_per_step"] / r["native"]["ms_per_step"], 2)
    else:
        rec["reference"] = "not available"
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
