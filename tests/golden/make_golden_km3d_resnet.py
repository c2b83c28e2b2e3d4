"""Golden vectors of KM3D / MonoFlex on the ResNet-18 CenterNet core: runs the UNMODIFIED reference (CPU, fp32) on the seeded synthetic
weights / inputs of visualdet3d_b200.synth and writes, next to this file:

  km3d_resnet_{96x320,192x640,384x1280}.npz   KM3D_example's detector (km3d_example_cfg, score_thr 0.1): features, head maps, detections
  monoflex_resnet_96x320.npz                  MonoFlex with Monoflex_example's commented-out ResNet-18 backbone (monoflex_resnet_cfg)
  km3d_resnet_keys.json / monoflex_resnet_keys.json   the reference's state_dict keys and shapes
  km3d_resnet_spread.npz                      [min, max] of every KM3D output entry over 8 torch seeds (method of make_golden_km3d_spread.py)

    python tests/golden/make_golden_km3d_resnet.py

KM3D_example names no backbone.  The reference's build_backbone then builds a ResNet, but its KM3DCore reads backbone_arguments['name']
itself (KM3D_core.py:16) and raises KeyError, so the reference is built here with name='resnet' spelled out: the same network and the
same state_dict keys the native KM3DCoreP builds from the name-less config.
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle"))
sys.path.insert(0, os.path.dirname(HERE))                 # tests/: centernet_resnet_oracle
import refload  # noqa: E402
from make_golden import flatten_fixture, subsample, to_edict  # noqa: E402
from visualdet3d_b200 import synth  # noqa: E402

N_SEEDS = 8
KM3D_CASES = [(96, 320, 2), (192, 640, 1), (384, 1280, 1)]


def cfgs(kind):
    """(native cfg, the cfg the reference is built from)"""
    from visualdet3d_b200.detectors.centernet import km3d_example_cfg, monoflex_resnet_cfg
    cfg = km3d_example_cfg(score_thr=0.1) if kind == "KM3D" else monoflex_resnet_cfg()
    ref_cfg = to_edict(json.loads(json.dumps(cfg)))
    ref_cfg.backbone.name = "resnet"
    return cfg, ref_cfg


def build_reference(kind, seed=0):
    refload.load_reference()
    from visualDet3D.networks.utils.registry import DETECTOR_DICT
    cfg, ref_cfg = cfgs(kind)
    torch.manual_seed(0)
    model = DETECTOR_DICT[kind](ref_cfg)
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    sd = synth.synth_state_dict(shapes, seed)
    missing = model.load_state_dict(sd, strict=False)
    print(kind, "missing:", missing.missing_keys, "unexpected:", missing.unexpected_keys)
    model.eval()
    return model, cfg, shapes, sd


def gen(kind, cases, seed=0):
    model, cfg, shapes, sd = build_reference(kind, seed)
    prefix = f"{kind.lower()}_resnet"
    with open(os.path.join(HERE, prefix + "_keys.json"), "w") as f:
        json.dump({k: list(v) for k, v in shapes.items()}, f, indent=0)
    import centernet_resnet_oracle as ro
    for (H, W, B) in cases:
        img, P2 = synth.synth_mono_inputs(B, H, W, seed=1)
        stages = {}
        hooks = [model.core.register_forward_hook(lambda m, i, o: stages.setdefault("features", []).append(o.detach().clone())),
                 model.bbox_head.register_forward_hook(
                     lambda m, i, o: stages.setdefault("heads", []).append({k: v.detach().clone() for k, v in o.items()}))]
        fix, outs = {}, []
        with torch.no_grad():
            for b in range(B):
                outs.append(model([img[b:b + 1], P2[b:b + 1]]))
        for h in hooks:
            h.remove()
        for b in range(B):
            s, bb, ci = outs[b]
            fix[f"scores_{b}"], fix[f"bboxes_{b}"], fix[f"cls_{b}"] = s.numpy(), bb.numpy(), ci.numpy()
            print(f"{kind}-ResNet {H}x{W} image {b}: {len(s)} detections")
        fix["features"] = subsample(torch.cat(stages["features"], 0))
        for n in cfg["head"]["layer_cfg"]["head_dict"]:
            fix["head_" + n] = subsample(torch.cat([x[n] for x in stages["heads"]], 0))
        fix["meta"] = np.array([H, W, B, seed], dtype=np.int64)
        np.savez_compressed(os.path.join(HERE, f"{prefix}_{H}x{W}.npz"), **flatten_fixture(fix))
        # immediate pin of the oracle (tests/centernet_resnet_oracle.py; also asserted by tests/test_km3d_resnet_cpu.py)
        st = {}
        o = (ro.km3d_forward if kind == "KM3D" else ro.monoflex_forward)(sd, img, P2, cfg, st)
        for b in range(B):
            same = len(o[b][0]) == len(outs[b][0])
            print("  oracle vs ref image", b, "n", len(o[b][0]), len(outs[b][0]),
                  "max|dbox|", float((o[b][1] - outs[b][1]).abs().max()) if same and len(o[b][0]) else None)
        print("  features max abs diff", float(np.abs(fix["features"]["samples"] - subsample(st["features"])["samples"]).max()),
              "absmean", fix["features"]["abssum"] / np.prod(fix["features"]["shape"]))
    return model


def gen_spread(model, seed=0):
    """The reference's own run-to-run spread (gen_position's randn * 1e-8 jitter of A^T A, rtm3d_utils.py:439-449)."""
    out = {"n_seeds": np.int64(N_SEEDS)}
    for (H, W, B) in KM3D_CASES:
        img, P2 = synth.synth_mono_inputs(B, H, W, seed=1)
        for b in range(B):
            runs = []
            for s in range(N_SEEDS):
                torch.manual_seed(1000 + s)
                with torch.no_grad():
                    sc, bb, ci = model([img[b:b + 1], P2[b:b + 1]])
                runs.append((sc.numpy().copy(), bb.numpy().copy(), ci.numpy().copy()))
            assert all(np.array_equal(r[2], runs[0][2]) and np.array_equal(r[0], runs[0][0]) for r in runs), "scores / classes must not depend on the jitter"
            bbs = np.stack([r[1] for r in runs]).astype(np.float64)
            lo, hi = bbs.min(0), bbs.max(0)
            tag = f"{H}x{W}_{b}"
            out[f"{tag}/min"], out[f"{tag}/max"] = lo.astype(np.float32), hi.astype(np.float32)
            out[f"{tag}/scores"] = runs[0][0]
            print(f"KM3D-ResNet {tag}: K={bbs.shape[1]}  max spread per column:", np.array2string((hi - lo).max(0), precision=2))
    np.savez_compressed(os.path.join(HERE, "km3d_resnet_spread.npz"), **out)


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    m = gen("KM3D", KM3D_CASES)
    gen_spread(m)
    gen("MonoFlex", [(96, 320, 2)])
