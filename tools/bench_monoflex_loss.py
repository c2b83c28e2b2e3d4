"""Time the MonoFlex head's training loss, forward + backward, native (visualdet3d_b200/monoflex_loss.py) against the reference's
`MonoFlexHead.loss` on the same GPU, at the Monoflex_example training shape: B = 8, 384x1280 images (96x320 maps), 3 classes, K = 32,
the targets of tests/golden/monoflex_loss.npz case a (4..12 objects per image).  Reports ms per step (host clock around steps ending in a
device synchronise: the reference's loss is host-bound), and from one profiled step each: kernel launches, device-to-host copies and
host synchronisations.  The reference arm runs under `torch.device("cuda")`: its _gather_output indexes a host arange with the device
reg_mask, which current torch refuses.  Prints the card's name, power limit and max SM clock; writes nothing.

    python tools/bench_monoflex_loss.py [--steps 50] [--warmup 10]
The reference arm needs the reference package (oracle/_ref/visualDet3D or the reference tree); without it only the native arm runs."""
import argparse
import importlib.util
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402
from bench_common import card, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    import refload
    from conftest import load_fixture
    from visualdet3d_b200 import _lib, monoflex_loss
    spec = importlib.util.spec_from_file_location("gen", os.path.join(ROOT, "tests", "golden", "make_golden_monoflex_loss.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    fx = load_fixture("monoflex_loss")["a"]
    out = {k: v.cuda().requires_grad_(True) for k, v in gen.head_outputs(fx).items()}
    ann = {k: v.cuda() for k, v in gen.annotations(fx).items()}
    ann["reg_mask"] = ann["reg_mask"].bool()
    P2 = torch.from_numpy(fx["P2"]).cuda()
    rec = dict(card=card(), torch=torch.__version__, steps=args.steps, warmup=args.warmup,
               B=int(fx["B"]), C=int(fx["C"]), H=int(fx["H"]), W=int(fx["W"]), K=int(fx["K"]), objects=int(fx["reg_mask"].sum()))

    def native():
        for t in out.values():
            t.grad = None
        loss, _ = monoflex_loss.monoflex_head_loss(out, ann, P2)
        loss.backward()

    rec["native"] = timed(native, args.steps, args.warmup)
    _lib.launch_count_reset()
    native()
    torch.cuda.synchronize()
    rec["native"]["native_launches"] = _lib.launch_count()
    if refload.available():
        from visualdet3d_b200.ops import dcn, iou3d
        refload.load_reference(device="cuda", dcn_ext=dcn, iou3d_ext=iou3d)
        from visualDet3D.networks.heads.monoflex_head import MonoFlexHead
        from visualdet3d_b200.detectors import monoflex_cfg
        head = MonoFlexHead(**refload.to_edict(dict(monoflex_cfg().head))).cuda().train()

        def reference():
            for t in out.values():
                t.grad = None
            with torch.device("cuda"):        # _gather_output indexes a host arange with the device reg_mask: made on the device
                loss, _ = head.loss(out, dict(ann), dict(P2=P2, epoch=0))
            loss.backward()

        rec["reference"] = timed(reference, max(1, args.steps // 5), max(1, args.warmup // 5))
        rec["speedup"] = round(rec["reference"]["ms_per_step"] / rec["native"]["ms_per_step"], 2)
    else:
        rec["reference"] = "not available"
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
