"""Golden vectors for visualdet3d_b200/monoflex_loss.py from the UNMODIFIED reference `MonoFlexHead.loss`
(R/networks/heads/monoflex_head.py:181-236) run forward and backward on the host through oracle/refload.py.
python tests/golden/make_golden_monoflex_loss.py  ->  tests/golden/monoflex_loss.npz

Targets are synthetic with the structure of KittiMonoFlexDataset._build_target (KM3D_dataset.py:346-520): Gaussian peaks of exactly 1
drawn by the reference's own gen_hm_radius, ind at the peak, the bin / residual rule of the dataset for rotbin / rotres, zero padding
rows.  Head outputs come from `synth.monoflex_head_outputs(seed)` plus the per-row edits stored with the case; the seed is redrawn until
no input lies within 1e-6 of a point where the loss is not differentiable (|pred - target| = 0, a clamp bound, a max / min tie, a
keypoint height of 0), except the edits placed there on purpose.

Cases:
  a  the Monoflex_example head at its training shape: B = 8, 96x320 maps (384x1280 images), 3 classes, K = 32, 4..12 objects per image
  b  edge batch, B = 4 at 24x80, K = 16: image 0 without objects; image 1 with two objects on one pixel, an object whose keypoint heights
     are all <= 0, mixed kp_detph_mask, rotbin rows with both and with neither bin set, a padding row with rotbin set, hps_mask partly
     0, depths on both sides of 5; image 2 whose heatmap has no exact 1; image 3 with uncertainties beyond both ends of the range
  c  no object anywhere and no gt == 1, B = 2 at 24x80, K = 8, some padding rows with hps_mask and rotbin set: the reference raises in
     _gather_output, so the fixture holds what its own static _neg_loss / _RegWeightedL1Loss / _RotLoss give (and their gradients); the
     six gathered terms are expected to be 0

Stored per case: sizes, seed, the targets (hm sparsely), P2, the edits, the sha256 of the nine maps, the nine terms and the total, and
the gradient of the total: for the eight gathered maps every nonzero element; for hm every pixel where the target is > 0 and a strided
sample; each gradient's max |.|.
"""
import hashlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, ROOT)
import refload  # noqa: E402
from visualdet3d_b200 import synth  # noqa: E402
from visualdet3d_b200.monoflex_loss import MAPS, TERMS  # noqa: E402

CASES = {
    "a": dict(B=8, C=3, H=96, W=320, K=32, seed=21, n_obj=(4, 12)),
    "b": dict(B=4, C=3, H=24, W=80, K=16, seed=22, n_obj=(3, 5)),
    "c": dict(B=2, C=3, H=24, W=80, K=8, seed=23, n_obj=(0, 0)),
}
HM_SAMPLE_STRIDE = 97
MARGIN = 1e-6


def sha(t: torch.Tensor) -> str:
    return hashlib.sha256(np.ascontiguousarray(t.detach().cpu().numpy().astype(np.float32)).tobytes()).hexdigest()


def maps_sha(out) -> str:
    h = hashlib.sha256()
    for name, _ in MAPS:
        h.update(sha(out[name]).encode())
    return h.hexdigest()


def head_outputs(fx):
    """The nine maps of a case: synth.monoflex_head_outputs(seed) and the stored edits at the rows' pixels (flip the sign of every
    keypoint y channel: all keypoint heights <= 0; set the four uncertainties)."""
    B, C, H, W = (int(fx[k]) for k in ("B", "C", "H", "W"))
    out = synth.monoflex_head_outputs(B, C, H, W, seed=int(fx["seed"]))
    ind = fx["ind"]
    for b, k in fx["flip_kp"].reshape(-1, 2):
        y, x = divmod(int(ind[b, k]), W)
        out["hps"][b, 1::2, y, x] *= -1
    for row in fx["unc_edit"].reshape(-1, 6):
        b, k = int(row[0]), int(row[1])
        y, x = divmod(int(ind[b, k]), W)
        out["depth_uncertainty"][b, 0, y, x] = float(row[2])
        out["corner_uncertainty"][b, :, y, x] = torch.from_numpy(row[3:6].astype(np.float32))
    return out


def hm_target(fx):
    B, C, H, W = (int(fx[k]) for k in ("B", "C", "H", "W"))
    hm = np.zeros(B * C * H * W, dtype=np.float32)
    hm[fx["hm_idx"]] = fx["hm_val"]
    return torch.from_numpy(hm.reshape(B, C, H, W))


def annotations(fx):
    """The reference's annotation dict of a case (dtypes of KittiMonoFlexDataset's collate: masks uint8, ind / rotbin int64)."""
    ann = dict(hm=hm_target(fx))
    for k in ("ind", "reg_mask", "hps", "hps_mask", "dep", "rotbin", "rotres", "bboxes2d_target", "dim", "reg", "kp_detph_mask"):
        ann[k] = torch.from_numpy(np.ascontiguousarray(fx[k]))
    return ann


def draw_targets(name, case, rng):
    from visualDet3D.networks.utils.rtm3d_utils import gen_hm_radius
    B, C, H, W, K = case["B"], case["C"], case["H"], case["W"], case["K"]
    hm = np.zeros((B, C, H, W), dtype=np.float32)
    t = dict(ind=np.zeros((B, K), np.int64), reg_mask=np.zeros((B, K), np.uint8), hps=np.zeros((B, K, 20), np.float32),
             hps_mask=np.zeros((B, K, 20), np.uint8), dep=np.zeros((B, K, 1), np.float32), rotbin=np.zeros((B, K, 2), np.int64),
             rotres=np.zeros((B, K, 2), np.float32), bboxes2d_target=np.zeros((B, K, 4), np.float32),
             dim=np.zeros((B, K, 3), np.float32), reg=np.zeros((B, K, 2), np.float32), kp_detph_mask=np.zeros((B, K, 3), np.float32))
    flip_kp, unc_edit = [], []
    for b in range(B):
        n = rng.randint(case["n_obj"][0], case["n_obj"][1] + 1)
        if name == "b" and b == 0:
            n = 0
        for k in range(n):
            cx, cy = rng.randint(0, W), rng.randint(0, H)
            if name == "b" and b == 1 and k == 1:
                cx, cy = int(t["ind"][b, 0] % W), int(t["ind"][b, 0] // W)           # the same pixel as row 0
            cls = rng.randint(C)
            gen_hm_radius(hm[b, cls], (cx, cy), rng.randint(1, 4))
            t["ind"][b, k] = cy * W + cx
            t["reg_mask"][b, k] = 1
            t["hps"][b, k] = rng.uniform(-10, 10, 20)
            t["hps_mask"][b, k] = 1
            t["dep"][b, k] = rng.uniform(3.0, 60.0)
            alpha = rng.uniform(-np.pi, np.pi)
            if np.sin(alpha) < 0.5:
                t["rotbin"][b, k, 0], t["rotres"][b, k, 0] = 1, alpha + 0.5 * np.pi
            if np.sin(alpha) > -0.5:
                t["rotbin"][b, k, 1], t["rotres"][b, k, 1] = 1, alpha - 0.5 * np.pi
            t["bboxes2d_target"][b, k] = rng.uniform(1.0, 12.0, 4)
            t["dim"][b, k] = rng.uniform(1.0, 4.0, 3)
            t["reg"][b, k] = rng.uniform(0.0, 1.0, 2)
            t["kp_detph_mask"][b, k] = 1.0
        if name == "b" and b == 1:
            t["hps_mask"][b, 2, 6:14] = 0
            t["kp_detph_mask"][b, 1] = [1.0, 0.0, 1.0]
            t["kp_detph_mask"][b, 2] = [0.0, 0.0, 0.0]
            t["dep"][b, 0], t["dep"][b, 1] = 3.5, 40.0
            t["rotbin"][b, 0], t["rotres"][b, 0] = [1, 1], [0.3, -0.4]
            t["rotbin"][b, 2], t["rotres"][b, 2] = [0, 0], [0.0, 0.0]
            flip_kp.append((b, 2))
            t["rotbin"][b, K - 1], t["rotres"][b, K - 1] = [0, 1], [0.0, 0.7]                    # a padding row with rotbin set
        if name == "b" and b == 2:
            hm[b] *= 0.75                                                                         # no exact 1
        if name == "b" and b == 3:
            unc_edit.append((b, 0, 12.0, -12.5, 0.5, 11.0))
            unc_edit.append((b, 1, -11.0, 13.0, -10.5, 2.0))
        if name == "c":
            for k in (1, 4):                                                                       # padding rows with hps_mask / rotbin
                t["ind"][b, k] = rng.randint(0, H * W)
                t["hps"][b, k] = rng.uniform(-10, 10, 20)
                t["hps_mask"][b, k, :12] = 1
                t["dep"][b, k] = rng.uniform(3.0, 60.0)
                t["rotbin"][b, k] = [1, 0]
                t["rotres"][b, k] = [rng.uniform(-1, 1), 0.0]
            hm[b, b % C, 5:8, 10:13] = 0.5
    if name == "c":
        assert not (hm == 1).any()
    idx = np.flatnonzero(hm.reshape(-1) > 0)
    return t, dict(hm_idx=idx.astype(np.int64), hm_val=hm.reshape(-1)[idx]), np.array(flip_kp, np.int64).reshape(-1, 2), \
        np.array(unc_edit, np.float64).reshape(-1, 6)


def away(x, points, scale=1.0):
    x = np.asarray(x, np.float64)
    return all(np.all(np.abs(x - p) > MARGIN * max(scale, abs(p))) for p in points)


def inputs_ok(fx, out, P2) -> bool:
    """No gathered quantity within MARGIN of a point where the loss is not differentiable (the edited rows' heights and uncertainties
    sit far beyond theirs on purpose)."""
    B, W = int(fx["B"]), int(fx["W"])
    g = lambda name, b, k: out[name][b, :, int(fx["ind"][b, k]) // W, int(fx["ind"][b, k]) % W].numpy().astype(np.float64)  # noqa: E731
    for b in range(B):
        for k in range(int(fx["K"])):
            if fx["hps_mask"][b, k].any() and not away((g("hps", b, k) - fx["hps"][b, k])[fx["hps_mask"][b, k] > 0], [0.0]):
                return False
            for j in range(2):
                if fx["rotbin"][b, k, j]:
                    o = g("rot", b, k)
                    r = float(fx["rotres"][b, k, j])
                    if not away([o[4 * j + 2] - np.sin(r), o[4 * j + 3] - np.cos(r)], [0.0, 1.0, -1.0]):
                        return False
            if not fx["reg_mask"][b, k]:
                continue
            o, q = g("bbox2d", b, k), fx["bboxes2d_target"][b, k].astype(np.float64)
            if not away(o - q, [0.0]) or not away([min(o[2], q[2]) + min(o[0], q[0]), min(o[3], q[3]) + min(o[1], q[1])], [0.0]):
                return False
            if not away(g("dim", b, k) - fx["dim"][b, k], [0.0]) or not away(g("reg", b, k) - fx["reg"][b, k], [0.0]):
                return False
            dep = float(fx["dep"][b, k, 0])
            if not away(np.exp(-g("depth", b, k)) - dep, [0.0], dep):
                return False
            u = np.concatenate([g("depth_uncertainty", b, k), g("corner_uncertainty", b, k)])
            if not away(u, [-10.0, 10.0]):
                return False
            y = g("hps", b, k)[1::2]
            ht = np.array([y[8] - y[9], y[7] - y[0], y[3] - y[4], y[2] - y[1], y[6] - y[5]])
            if not away(ht, [0.0]):
                return False
            if (ht > 0).all():
                fh = float(P2[b, 0, 0]) * g("dim", b, k)[1]
                d = fh / (ht * 4 + 1e-8)
                kd = np.array([d[0], (d[1] + d[2]) / 2, (d[3] + d[4]) / 2])
                if not away(kd, [0.1, 100.0]) or not away(kd - dep, [0.0], dep):
                    return False
    return True


def run_reference(name, fx, out, P2):
    from visualDet3D.networks.heads.monoflex_head import MonoFlexHead
    C, K = int(fx["C"]), int(fx["K"])
    for t in out.values():
        t.requires_grad_(True)
    ann = annotations(fx)
    if name == "c":
        hm = MonoFlexHead._neg_loss(out["hm"], ann["hm"])
        hp = MonoFlexHead._RegWeightedL1Loss(out["hps"], ann["hps_mask"], ann["ind"], ann["hps"], ann["dep"].clone())
        rot = MonoFlexHead._RotLoss(out["rot"], ann["reg_mask"].bool(), ann["ind"], ann["rotbin"], ann["rotres"])
        zero = torch.zeros(())
        stats = dict(zip(TERMS, (hm, hp, zero, zero, zero, zero, zero, rot, zero)))
        total = 0
        for key, w in zip(TERMS, (1, 1, 1, 0.5, 1, 1, 0.2, 1.0, 0.2)):
            total = total + stats[key] * w
    else:
        layer = dict(input_features=8, head_features=8, head_dict={n: (C if ch is None else ch) for n, ch in MAPS})
        head = MonoFlexHead(num_classes=C, num_joints=9, max_objects=K, layer_cfg=refload.to_edict(layer),
                            loss_cfg=refload.to_edict(dict(gamma=2.0, output_w=float(fx["W"]))), test_cfg=refload.to_edict(dict(score_thr=0.1)))
        total, stats = head.loss(out, ann, dict(P2=P2, epoch=0))
    total.backward()
    return total, stats


def run_case(name, case):
    rng = np.random.RandomState(case["seed"])
    t, hm, flip_kp, unc_edit = draw_targets(name, case, rng)
    B, H, W = case["B"], case["H"], case["W"]
    P2, _ = synth.synth_P2(B, H * 4, W * 4)
    fx = dict(case, **t, **hm, flip_kp=flip_kp, unc_edit=unc_edit, P2=P2.numpy())
    fx.pop("n_obj")
    seed = case["seed"] * 1000
    while True:
        fx["seed"] = seed
        out = head_outputs(fx)
        if inputs_ok(fx, out, P2):
            break
        seed += 1
    fx["maps_sha"] = np.array(maps_sha(out))
    total, stats = run_reference(name, fx, out, P2)
    fx["terms"] = np.array([float(stats[k].detach()) for k in TERMS], dtype=np.float32)
    fx["total"] = np.float32(float(total.detach()))
    for mname, _ in MAPS:
        gr = out[mname].grad
        gr = np.zeros(tuple(out[mname].shape), np.float32) if gr is None else gr.numpy()
        flat = gr.reshape(-1)
        if mname == "hm":
            idx = np.union1d(fx["hm_idx"], np.arange(0, flat.size, HM_SAMPLE_STRIDE))
        else:
            idx = np.flatnonzero(flat)
        fx[f"grad_{mname}_idx"] = idx.astype(np.int64)
        fx[f"grad_{mname}"] = flat[idx]
        fx[f"grad_{mname}_max"] = np.float32(np.abs(flat).max())
    print(f"case {name}: seed={seed} terms={dict(zip(TERMS, fx['terms'].tolist()))} total={float(fx['total']):.6g} "
          f"objects={int(fx['reg_mask'].sum())}")
    return fx


def main():
    refload.load_reference()
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    fix = {}
    for name, case in CASES.items():
        for k, v in run_case(name, case).items():
            fix[f"{name}/{k}"] = np.asarray(v)
    path = os.path.join(HERE, "monoflex_loss.npz")
    np.savez_compressed(path, **fix)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
