"""Secondary measurements (BASELINE.json configs[2], configs[3] and the configs[0] plumbing case on the GPU): device-resident
forward rate of the other detectors of the hot path, CUDA events, inputs larger than L2 or L2 flushed by the step itself.
usage: python tools/bench_detectors.py [steps] [name,name]   -> one JSON line per detector"""
import json, os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from visualdet3d_b200 import synth, _lib
from visualdet3d_b200.detectors import build_synthetic_mono3d, build_synthetic_monoflex

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
only = set(sys.argv[2].split(",")) if len(sys.argv) > 2 else None
CASES = [("Yolo3D", "configs[0] shape on the GPU: Yolo3D ResNet-18 (DCNv2 head)", 1, 288, 1280, lambda: build_synthetic_mono3d("Yolo3D", seed=0, depth=18)[0]),
         ("Yolo3D-b8", "Yolo3D ResNet-18 (DCNv2 head), batch 8", 8, 288, 1280, lambda: build_synthetic_mono3d("Yolo3D", seed=0, depth=18)[0]),
         ("GroundAwareYolo3D", "configs[2]: Ground-aware Mono3D (GAC head, ResNet-101), batch 8 mono 288x1280", 8, 288, 1280,
          lambda: build_synthetic_mono3d("GroundAwareYolo3D", seed=0)[0]),
         ("MonoFlex", "configs[3]: MonoFlex DLA-34 + DCNv2, batch 8, 384x1280", 8, 384, 1280, lambda: build_synthetic_monoflex(seed=0)[0]),
         ("KM3D", "configs[3]: KM3D DLA-34 + DCNv2, batch 8, 384x1280", 8, 384, 1280, lambda: build_synthetic_monoflex(seed=0, name="KM3D")[0]),
         ("KM3D-resnet18", "KM3D_example: ResNet-18 + transposed-conv up-sampling, batch 8, 384x1280", 8, 384, 1280,
          lambda: build_synthetic_monoflex(seed=0, name="KM3D", backbone="resnet18")[0])]
for name, desc, B, H, W, mk in CASES:
    if only and name not in only:
        continue
    try:
        det = mk().cuda().eval()
        img, P2 = synth.synth_mono_inputs(B, H, W, seed=1)
        img, P2 = img.cuda(), P2.cuda()
        with torch.no_grad():
            for _ in range(3):
                det.launch(img, P2)
            torch.cuda.synchronize()
            _lib.launch_count_reset()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                det.launch(img, P2)
            e1.record()
            torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / steps
        print(json.dumps({"detector": name, "workload": desc, "batch": B, "ms_per_step": ms, "images_per_s": B / ms * 1e3,
                          "gpu_launches_per_step": _lib.launch_count() / steps, "steps": steps, "data": "synthetic", "dtype": "f32"}), flush=True)
        del det
        torch.cuda.empty_cache()
    except Exception as ex:
        print(json.dumps({"detector": name, "error": repr(ex)[:300]}), flush=True)
