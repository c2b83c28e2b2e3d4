"""Golden vectors for visualdet3d_b200/km3d_loss.py from the UNMODIFIED reference `KM3DHead.loss` (R/networks/heads/km3d_head.py:316-351)
run forward and backward on the host through oracle/refload.py.
python tests/golden/make_golden_km3d_loss.py  ->  tests/golden/km3d_loss.npz

The only CUDA pieces of the reference loss are inside boxes_iou3d_gpu (R/lib/ops/iou3d/iou3d.py:37-71); while the reference runs they get
host stand-ins: boxes_overlap_bev_gpu becomes oracle/torch_port.rotated_overlap_bev (an independent float64 algorithm) on the diagonal --
the only entries Position_loss reads; the others stay 0 -- and torch.cuda.FloatTensor a host zero allocation.  torch is seeded for the
solve's randn jitter.

Targets follow KittiRTM3DDataset._build_target (KM3D_dataset.py:55-221): boxes in front of the camera; hps are the 8 corners (in the
order gen_position's equations use: corner j = location + (B_j, B_j+1, C_j)) and the centre projected through P2 to the 1/4 map,
relative to the centre pixel (P2 with fy = fx and no y / z translation: gen_position assumes both); peaks of exactly 1 drawn by the reference's gen_hm_radius (hm at the centre, hm_hp at each keypoint);
hp_ind / hp_offset / hp_mask per keypoint inside the map; the dataset's bin / residual rule for rotbin / rotres.  Head outputs are
seeded uniform maps with, at each object's pixel, keypoints, dims and rotation bins written near the targets (the stored edits), so the
solved positions land near `location` and most IoUs lie strictly inside (0, 1).

Cases:
  a  the KM3D_example head at its training shape: B = 8, 96x320 maps, 3 classes, K = 32, 4..12 objects per image
  b  edge batch, B = 4 at 24x80, K = 16: image 0 without objects; image 1 with two objects on one pixel (so colliding hp_ind), a reg_mask
     row whose hps_mask sums to 14, a negative predicted dim, rotbin rows with both bins and with neither, a padding row with rotbin set,
     dep on both sides of 5, a disjoint (IoU 0) pair; image 2 whose predicted rot_y wraps past -pi and whose hm has no exact 1; image 3
     whose predicted rot_y wraps past +pi and whose hm_hp has no exact 1
  c  no object anywhere (mask_num = 0), B = 2 at 24x80, K = 8
  d  objects, but no exact 1 anywhere in hm while hm_hp has its peaks (hm's num_pos == 0, hm_hp's > 0), B = 2 at 24x80, K = 8
  e  the reverse: hm_hp without an exact 1 anywhere, hm with its peaks
Totals at epochs 0, 37 and 100 (= rampup_length); terms and gradients at epoch 37.  Per case also coor_loss restated in float64 without
jitter (coor_loss64) with its hps / dim gradients, and how far the float32 reference's coor_loss and gradients lie from it: the float32
scatter the reference itself has, which bounds how closely any float32 implementation can match it.
"""
import contextlib
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
from visualdet3d_b200.km3d_loss import MAPS, TERMS  # noqa: E402

CASES = {
    "a": dict(B=8, C=3, H=96, W=320, K=32, seed=31, n_obj=(4, 12)),
    "b": dict(B=4, C=3, H=24, W=80, K=16, seed=32, n_obj=(2, 4)),
    "c": dict(B=2, C=3, H=24, W=80, K=8, seed=33, n_obj=(0, 0)),
    "d": dict(B=2, C=3, H=24, W=80, K=8, seed=34, n_obj=(2, 3)),
    "e": dict(B=2, C=3, H=24, W=80, K=8, seed=35, n_obj=(2, 3)),
}
EPOCHS = (0, 37, 100)
GRAD_EPOCH = 37
RAMPUP = 100
HM_SAMPLE_STRIDE = 97
ANN_KEYS = ("ind", "reg_mask", "hps", "hps_mask", "dep", "rotbin", "rotres", "wh", "dim", "reg", "hp_ind", "hp_mask", "hp_offset",
            "location", "ori")
# gen_position's corner offsets: x = sxl * l/2 cos + sxw * w/2 sin ... (rtm3d_utils.py:402-434, corners j = 0..7)
SXL = np.array([-1, -1, -1, 1, 1, 1, 1, -1.0])
SXW = np.array([-1, 1, 1, 1, 1, -1, -1, -1.0])
SY = np.array([-1, -1, 1, 1, -1, -1, 1, 1.0])
SCL = np.array([1, 1, 1, -1, -1, -1, -1, 1.0])
SCW = np.array([-1, 1, 1, 1, 1, -1, -1, -1.0])


def sha(t: torch.Tensor) -> str:
    return hashlib.sha256(np.ascontiguousarray(t.detach().cpu().numpy().astype(np.float32)).tobytes()).hexdigest()


def maps_sha(out) -> str:
    h = hashlib.sha256()
    for name, _ in MAPS:
        h.update(sha(out[name]).encode())
    return h.hexdigest()


def head_outputs(fx):
    """The nine maps of a case: seeded uniform maps (hm / hm_hp logits on a 1/8 grid over [-6, 6], away from the focal loss's cuts) and
    the stored edits at the object rows' pixels (rows in order, so a later row on the same pixel wins)."""
    B, C, H, W = (int(fx[k]) for k in ("B", "C", "H", "W"))
    rng = np.random.RandomState(int(fx["seed"]))
    u = lambda lo, hi, ch: rng.uniform(lo, hi, size=(B, ch, H, W)).astype(np.float32)  # noqa: E731
    out = dict(hm=(rng.randint(-48, 49, size=(B, C, H, W)) / 8).astype(np.float32), wh=u(1.0, 20.0, 2), hps=u(-8.0, 8.0, 18),
               rot=u(-2.0, 2.0, 8), dim=u(1.0, 4.0, 3), prob=u(-3.0, 3.0, 1), reg=u(0.0, 1.0, 2),
               hm_hp=(rng.randint(-48, 49, size=(B, 9, H, W)) / 8).astype(np.float32), hp_offset=u(0.0, 1.0, 2))
    for row in fx["edits"]:
        b, k = int(row[0]), int(row[1])
        y, x = divmod(int(fx["ind"][b, k]), W)
        out["hps"][b, :, y, x] = row[2:20]
        out["rot"][b, :, y, x] = row[20:28]
        out["dim"][b, :, y, x] = row[28:31]
    return {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in out.items()}


def dense(fx, key, shape):
    a = np.zeros(int(np.prod(shape)), dtype=np.float32)
    a[fx[key + "_idx"]] = fx[key + "_val"]
    return torch.from_numpy(a.reshape(shape))


def annotations(fx):
    """The reference's annotation dict of a case (dtypes of the dataset's collate: masks uint8, ind / hp_ind / rotbin int64)."""
    B, C, H, W = (int(fx[k]) for k in ("B", "C", "H", "W"))
    ann = dict(hm=dense(fx, "hm", (B, C, H, W)), hm_hp=dense(fx, "hm_hp", (B, 9, H, W)))
    for k in ANN_KEYS:
        ann[k] = torch.from_numpy(np.array(fx[k]))                  # a copy: the reference rewrites dep in place
    return ann


def corners(X, Y, Z, w, h, l, ry):
    """The 8 corners and the centre in camera coordinates, in gen_position's keypoint order."""
    c, s = np.cos(ry), np.sin(ry)
    lc, ls, wc, ws, hh = l * 0.5 * c, l * 0.5 * s, w * 0.5 * c, w * 0.5 * s, h * 0.5
    pts = np.stack([X + SXL * lc + SXW * ws, Y + SY * hh, Z + SCL * ls + SCW * wc], 1)
    return np.concatenate([pts, [[X, Y, Z]]], 0)


def project(P, pts):
    hom = np.concatenate([pts, np.ones((len(pts), 1))], 1) @ P.T
    return hom[:, :2] / hom[:, 2:]


def wrap(a):
    return (a + np.pi) % (2 * np.pi) - np.pi


def draw_targets(name, case, P2, rng):
    from visualDet3D.networks.utils.rtm3d_utils import gen_hm_radius
    B, C, H, W, K = case["B"], case["C"], case["H"], case["W"], case["K"]
    hm = np.zeros((B, C, H, W), np.float32)
    hm_hp = np.zeros((B, 9, H, W), np.float32)
    t = dict(ind=np.zeros((B, K), np.int64), reg_mask=np.zeros((B, K), np.uint8), hps=np.zeros((B, K, 18), np.float32),
             hps_mask=np.zeros((B, K, 18), np.uint8), dep=np.zeros((B, K, 1), np.float32), rotbin=np.zeros((B, K, 2), np.int64),
             rotres=np.zeros((B, K, 2), np.float32), wh=np.zeros((B, K, 2), np.float32), dim=np.zeros((B, K, 3), np.float32),
             reg=np.zeros((B, K, 2), np.float32), hp_ind=np.zeros((B, K * 9), np.int64), hp_mask=np.zeros((B, K * 9), np.uint8),
             hp_offset=np.zeros((B, K * 9, 2), np.float32), location=np.zeros((B, K, 3), np.float32), ori=np.zeros((B, K, 1), np.float32))
    edits = []
    for b in range(B):
        P = P2[b].astype(np.float64)
        f, pcx = P[0, 0], P[0, 2]
        n = rng.randint(case["n_obj"][0], case["n_obj"][1] + 1)
        if name == "b":
            n = (0, 4, 2, 2)[b]
        for k in range(n):
            while True:
                Z = rng.uniform(10.0, 40.0)
                X, Y = rng.uniform(-0.4, 0.4) * Z, rng.uniform(0.5, 2.0)
                if name == "b" and b == 1 and k == 1:
                    X, Y, Z = t["location"][b, 0]                                   # the same pixel as row 0
                    X += 0.01
                w, h, l = rng.uniform(1.4, 2.0), rng.uniform(1.4, 1.8), rng.uniform(3.0, 4.5)
                u8 = project(P, np.array([[X, Y, Z]]))[0]
                alpha = rng.uniform(-np.pi, np.pi)
                if name == "b" and b == 2:
                    alpha = -np.pi + 0.02                                              # with the centre left of cx: rot_y < -pi
                if name == "b" and b == 3:
                    alpha = np.pi - 0.02                                               # with the centre right of cx: rot_y > pi
                ray = np.arctan2(u8[0] - pcx, f)
                if (name == "b" and b == 2 and ray > -0.1) or (name == "b" and b == 3 and ray < 0.1):
                    continue
                ry = wrap(alpha + ray)
                kp = project(P, corners(X, Y, Z, w, h, l, ry)) / 4
                ci = np.floor(kp[8]).astype(np.int64)
                if 0 <= ci[0] < W and 0 <= ci[1] < H:
                    break
            cls = rng.randint(C)
            radius = rng.randint(1, 4)
            gen_hm_radius(hm[b, cls], ci, radius)
            t["ind"][b, k] = ci[1] * W + ci[0]
            t["reg_mask"][b, k] = 1
            t["hps"][b, k] = (kp - ci).reshape(-1)
            t["hps_mask"][b, k] = 1
            t["dep"][b, k] = Z
            if np.sin(alpha) < 0.5:
                t["rotbin"][b, k, 0], t["rotres"][b, k, 0] = 1, alpha + 0.5 * np.pi
            if np.sin(alpha) > -0.5:
                t["rotbin"][b, k, 1], t["rotres"][b, k, 1] = 1, alpha - 0.5 * np.pi
            t["wh"][b, k] = rng.uniform(2.0, 20.0, 2)
            t["dim"][b, k] = (w, h, l)
            t["reg"][b, k] = rng.uniform(0.0, 1.0, 2)
            t["location"][b, k] = (X, Y, Z)
            t["ori"][b, k] = ry
            for j in range(9):
                vi = np.floor(kp[j]).astype(np.int64)
                if 0 <= vi[0] < W and 0 <= vi[1] < H:
                    gen_hm_radius(hm_hp[b, j], vi, radius)
                    t["hp_ind"][b, k * 9 + j] = vi[1] * W + vi[0]
                    t["hp_offset"][b, k * 9 + j] = kp[j] - vi
                    t["hp_mask"][b, k * 9 + j] = 1
            # predictions near the targets: keypoints, dims and the rotation bins of alpha (bin 1 for alpha < 0, else bin 2)
            noise = lambda n_: rng.choice([-1.0, 1.0], n_) * rng.uniform(0.01, 0.08, n_)  # noqa: E731
            rot = rng.uniform(-2.0, 2.0, 8)
            if alpha < 0:
                tt = alpha + 0.5 * np.pi
                rot[1], rot[5], rot[2], rot[3] = 1.0, -1.0, np.sin(tt) + noise(1)[0] * 0.1, np.cos(tt) + noise(1)[0] * 0.1
            else:
                tt = alpha - 0.5 * np.pi
                rot[1], rot[5], rot[6], rot[7] = -1.0, 1.0, np.sin(tt) + noise(1)[0] * 0.1, np.cos(tt) + noise(1)[0] * 0.1
            edits.append(np.concatenate([[b, k], t["hps"][b, k] + noise(18), rot, t["dim"][b, k] + noise(3)]))
        if name == "b" and b == 1:
            t["hps_mask"][b, 2, 14:] = 0                                   # sums to 14: no position / score for this row
            edits[-1][28] = -0.3                                          # row 3: a negative predicted dim
            t["dep"][b, 0] = 3.5                                         # dep below 5
            t["rotbin"][b, 0], t["rotres"][b, 0] = [1, 1], [0.3, -0.4]     # both bins
            t["rotbin"][b, 2], t["rotres"][b, 2] = [0, 0], [0.0, 0.0]      # neither
            t["rotbin"][b, K - 1], t["rotres"][b, K - 1] = [0, 1], [0.0, 0.7]   # a padding row with rotbin set
            t["location"][b, 1] += np.array([6.0, 0.0, 6.0], np.float32)  # a disjoint (IoU 0) pair
        if name == "b" and b == 2:
            hm[b] *= 0.75                                                  # hm without an exact 1 (hm_hp has them)
        if name == "b" and b == 3:
            hm_hp[b] *= 0.75                                               # hm_hp without an exact 1 (hm has them)
    if name == "d":
        hm *= 0.75                                                         # num_pos == 0 for hm only, batch-wide
    if name == "e":
        hm_hp *= 0.75                                                      # num_pos == 0 for hm_hp only, batch-wide
    fx = dict(t)
    for key, m in (("hm", hm), ("hm_hp", hm_hp)):
        idx = np.flatnonzero(m.reshape(-1) > 0)
        fx[key + "_idx"], fx[key + "_val"] = idx.astype(np.int64), m.reshape(-1)[idx]
    fx["edits"] = np.array(edits, np.float32).reshape(-1, 31)
    return fx


@contextlib.contextmanager
def host_iou3d():
    """boxes_iou3d_gpu's two CUDA pieces on the host (see the module docstring)."""
    import torch_port as tp
    from visualDet3D.networks.lib.ops.iou3d import iou3d as ref_iou3d

    def overlap(a, b, out):
        for i in range(min(len(a), len(b))):
            out[i, i] = tp.rotated_overlap_bev(a[i].numpy().astype(np.float64), b[i].numpy().astype(np.float64))

    saved = (ref_iou3d.boxes_overlap_bev_gpu, torch.cuda.FloatTensor)
    ref_iou3d.boxes_overlap_bev_gpu = overlap
    torch.cuda.FloatTensor = lambda size: torch.zeros(size)
    try:
        yield
    finally:
        ref_iou3d.boxes_overlap_bev_gpu, torch.cuda.FloatTensor = saved


def make_head(C, K, W):
    from visualDet3D.networks.heads.km3d_head import KM3DHead
    layer = dict(input_features=8, head_features=8, head_dict={n: (C if ch is None else ch) for n, ch in MAPS})
    return KM3DHead(num_classes=C, num_joints=9, max_objects=K, layer_cfg=refload.to_edict(layer),
                    loss_cfg=refload.to_edict(dict(gamma=2.0, output_w=W, rampup_length=RAMPUP)), test_cfg=refload.to_edict(dict(score_thr=0.1)))


def run_reference(fx, out, P2, epoch, backward):
    head = make_head(int(fx["C"]), int(fx["K"]), int(fx["W"]))
    torch.manual_seed(0)
    with host_iou3d():
        total, stats = head.loss(out, annotations(fx), dict(P2=P2, epoch=epoch))
    if backward:
        total.backward()
    return total, stats


def coor_loss64(fx, out, P2):
    """Position_loss's coor_loss (rtm3d_utils.py:242-290 with gen_position :314-455) restated in float64 throughout, with no jitter: the
    exact value the float32 reference (and the device) approximate.  out: the maps, float64 leaves for hps and dim."""
    B, W, K = int(fx["B"]), int(fx["W"]), int(fx["K"])
    ind = torch.from_numpy(np.array(fx["ind"]))
    gather = lambda m: m.permute(0, 2, 3, 1).reshape(B, -1, m.shape[1]).gather(1, ind[..., None].expand(B, K, m.shape[1]))  # noqa: E731
    hps, dim, rot = gather(out["hps"]), gather(out["dim"]), gather(out["rot"]).detach()
    cy = (ind.float() / W).int().double()                      # the reference's float32 division, then trunc
    cx = (ind % W).double()
    P = torch.from_numpy(np.array(fx["P2"])).double()[:, None]     # [B, 1, 3, 4]
    f, pcx, pcy = P[..., 0, 0], P[..., 0, 2], P[..., 1, 2]
    kx, ky = (hps[..., 0::2] + cx[..., None]) * 4, (hps[..., 1::2] + cy[..., None]) * 4
    alpha = torch.where(rot[..., 1] > rot[..., 5], torch.atan(rot[..., 2] / rot[..., 3]) - 0.5 * np.pi,
                        torch.atan(rot[..., 6] / rot[..., 7]) + 0.5 * np.pi)
    ry = alpha + torch.atan2(kx[..., 8] - pcx, f)
    ry = torch.where(ry > np.pi, ry - 2 * np.pi, ry)
    ry = torch.where(ry < -np.pi, ry + 2 * np.pi, ry)
    w, h, l = dim[..., 0:1], dim[..., 1:2], dim[..., 2:3]
    co, si = torch.cos(ry)[..., None], torch.sin(ry)[..., None]
    t = lambda v: torch.tensor(v, dtype=torch.float64)  # noqa: E731
    Bx = t(SXL) * l * 0.5 * co + t(SXW) * w * 0.5 * si
    By = t(SY) * h * 0.5
    Cc = t(SCL) * l * 0.5 * si + t(SCW) * w * 0.5 * co
    nx, ny = (kx[..., :8] - pcx[..., None]) / f[..., None], (ky[..., :8] - pcy[..., None]) / f[..., None]
    A = torch.zeros(B, K, 16, 3, dtype=torch.float64)
    A[..., 0::2, 0] = -1
    A[..., 1::2, 1] = -1
    A[..., 0::2, 2], A[..., 1::2, 2] = nx, ny
    b = torch.stack([Bx - nx * Cc, By - ny * Cc], -1).reshape(B, K, 16, 1)
    At = A.transpose(-1, -2)
    pos = torch.linalg.solve(At @ A, At @ b)[..., 0]
    pos = pos - torch.stack([P[..., 0, 3] / f, torch.zeros_like(f), torch.zeros_like(f)], -1)
    lm = (torch.from_numpy(np.array(fx["hps_mask"])).double().sum(2) > 15).double()
    loc = torch.from_numpy(np.array(fx["location"])).double()
    return ((pos - loc).norm(dim=2) * lm).sum() / (lm.sum() + 1)


def coor_scatter(fx, out, P2):
    """How far the float32 reference's coor_loss and its hps / dim gradients lie from the float64 restatement: relative for the value, of
    each map's total-gradient max for the gradients (the scale the GPU test compares at).  Also returns the float64 gradients."""
    o32 = {k: v.detach().clone().requires_grad_(True) for k, v in out.items()}
    head = make_head(int(fx["C"]), int(fx["K"]), int(fx["W"]))
    torch.manual_seed(0)
    with host_iou3d():
        c32, _, _ = head.position_loss(o32, annotations(fx), P2)
    c32.backward()
    o64 = {k: v.detach().double().requires_grad_(k in ("hps", "dim")) for k, v in out.items()}
    c64 = coor_loss64(fx, o64, P2)
    v32, v64 = float(c32.detach()), float(c64.detach())
    rec = dict(coor64=np.float64(v64), coor_ref_relerr=np.float64(abs(v32 - v64) / max(v64, 1e-30)))
    if c64.requires_grad:
        c64.backward()
    for m in ("hps", "dim"):
        g64 = np.zeros(tuple(out[m].shape)) if o64[m].grad is None else o64[m].grad.numpy()
        g32 = np.zeros(tuple(out[m].shape)) if o32[m].grad is None else o32[m].grad.numpy().astype(np.float64)
        gmax = float(fx[f"grad_{m}_max"])
        rec[f"pos_ref_err_{m}"] = np.float64(np.abs(g32 - g64).max() / gmax if gmax > 0 else 0.0)
        idx = np.flatnonzero(g64.reshape(-1))
        rec[f"pos64_{m}_idx"], rec[f"pos64_{m}"] = idx.astype(np.int64), g64.reshape(-1)[idx]
    return rec


def run_case(name, case):
    rng = np.random.RandomState(case["seed"])
    B, H, W = case["B"], case["H"], case["W"]
    P2, _ = synth.synth_P2(B, H * 4, W * 4)
    P2[:, 1, 1] = P2[:, 0, 0]                 # gen_position normalises both keypoint coordinates by P[0, 0]
    P2[:, 1:, 3] = 0.0                        # and compensates only P[0, 3]
    fx = dict(case, **draw_targets(name, case, P2.numpy(), rng), P2=P2.numpy())
    fx.pop("n_obj")
    fx["seed"] = case["seed"] * 1000
    out = head_outputs(fx)
    fx["maps_sha"] = np.array(maps_sha(out))
    for t in out.values():
        t.requires_grad_(True)
    fx["totals"] = np.array([float(run_reference(fx, {k: v.detach() for k, v in out.items()}, P2, e, False)[0]) for e in EPOCHS],
                            np.float32)
    total, stats = run_reference(fx, out, P2, GRAD_EPOCH, True)
    fx["terms"] = np.array([float(stats[k].detach()) for k in TERMS], dtype=np.float32)
    fx["total"] = np.float32(float(total.detach()))
    for mname, _ in MAPS:
        gr = out[mname].grad
        gr = np.zeros(tuple(out[mname].shape), np.float32) if gr is None else gr.numpy()
        flat = gr.reshape(-1)
        if mname in ("hm", "hm_hp"):
            idx = np.union1d(fx[mname + "_idx"], np.arange(0, flat.size, HM_SAMPLE_STRIDE))
        else:
            idx = np.flatnonzero(flat)
        fx[f"grad_{mname}_idx"] = idx.astype(np.int64)
        fx[f"grad_{mname}"] = flat[idx]
        fx[f"grad_{mname}_max"] = np.float32(np.abs(flat).max())
    fx.update(coor_scatter(fx, out, P2))
    print(f"case {name}: coor_loss float32 vs float64 {float(fx['coor_ref_relerr']):.2e}, hps / dim gradient "
          f"{float(fx['pos_ref_err_hps']):.2e} / {float(fx['pos_ref_err_dim']):.2e} of max")
    print(f"case {name}: terms={dict(zip(TERMS, fx['terms'].tolist()))} totals={fx['totals'].tolist()} objects={int(fx['reg_mask'].sum())}")
    return fx


def main():
    refload.load_reference()
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    fix = {}
    for name, case in CASES.items():
        for k, v in run_case(name, case).items():
            fix[f"{name}/{k}"] = np.asarray(v)
    path = os.path.join(HERE, "km3d_loss.npz")
    np.savez_compressed(path, **fix)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
