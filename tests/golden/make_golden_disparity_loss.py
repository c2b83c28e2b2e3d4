"""Golden vectors for visualdet3d_b200/disparity_loss.py from the UNMODIFIED reference disparity loss (DisparityLoss(max_disp).criterion,
i.e. StereoFocalLoss with LaplaceDisp2Prob, R/networks/heads/losses.py:122-135 and R/networks/lib/disparity_loss/*.py) run on the host
through oracle/refload.py: `DisparityLoss(max_disp).criterion(x, label.unsqueeze(1), variance=0.5)`, which is DisparityLoss.forward's body
without the label's `.cuda()`.
python tests/golden/make_golden_disparity_loss.py  ->  tests/golden/disparity_loss.npz

Cases (the logits are randn * 2 from a seeded torch.Generator; labels on the 1/16 grid from a seeded RandomState):
  a  the Stereo3D_example training shape: B=4, D=96, 72x320 maps; zero above a horizon row, sparse below it (about 23 % valid), values
     up to 140, so some lie at or above 96
  b  an edge batch at B=3, 8x48: an image with no valid pixel (only 0, 96, 200 and negative labels); labels exactly 0, 1/16, 1, 94.9375,
     95, 95.5, 95.9375, 96 and 200 in a row; a pixel whose logits are offset by +1000; a pixel with a +-60 logit spread
  c  a batch with no valid pixel at all (the reference's print branch: loss 0, gradient 0)
  d  DisparityLoss(64) with D=64, B=2, 36x160

The inputs are regenerated from their seeds by the tests (their sha256 is stored and checked), so the file holds: the reference's fp32
loss; the float64 restatement's loss (`restate`); the reference's gradient of the loss at a strided sample of the volume and at every
channel of the named pixels (the edge pixels of b, and pixels in the [max_disp - 1, max_disp) band); the gradient's max |.|; the number
of pixels with 0 < label < max_disp.
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

CASES = {
    "a": dict(B=4, D=96, H=72, W=320, seed=21, horizon=24, density=0.5, top=140.0, stride=997),
    "b": dict(B=3, D=96, H=8, W=48, seed=22, horizon=0, density=0.5, top=120.0, stride=7),
    "c": dict(B=2, D=96, H=8, W=40, seed=23, horizon=0, density=0.0, top=0.0, stride=7),
    "d": dict(B=2, D=64, H=36, W=160, seed=24, horizon=12, density=0.5, top=90.0, stride=499),
}
B_EDGE_ROW = (0.0, 1.0 / 16, 1.0, 94.9375, 95.0, 95.5, 95.9375, 96.0, 200.0)    # case b, image 1, row 2, columns 0..8
B_OFFSET_PIXEL = (1, 4, 5, 30.5)       # (image, y, x, label): logits + 1000
B_SPREAD_PIXEL = (1, 4, 6, 47.25)      # logits uniform in [-60, 60]
N_BAND = 8                             # band pixels named per case


def sha(t: torch.Tensor) -> str:
    return hashlib.sha256(np.ascontiguousarray(t.detach().cpu().numpy().astype(np.float32)).tobytes()).hexdigest()


def inputs(name: str):
    """(x [B, D, H, W], label [B, H, W]) float32 on the host, regenerated from the case's seed."""
    c = CASES[name]
    B, D, H, W = c["B"], c["D"], c["H"], c["W"]
    g = torch.Generator().manual_seed(c["seed"])
    x = torch.randn(B, D, H, W, generator=g) * 2
    rng = np.random.RandomState(c["seed"])
    lab = np.zeros((B, H, W), dtype=np.float32)
    if c["density"] > 0:
        valid = rng.uniform(size=(B, H, W)) < c["density"]
        valid[:, :c["horizon"]] = False
        vals = np.round(rng.uniform(0.0, c["top"], size=(B, H, W)) * 16) / 16
        lab[valid] = vals[valid]
    if name == "b":
        lab[0] = 0.0
        lab[0, 1, 3], lab[0, 5, 7], lab[0, 6, 20], lab[0, 2, 9] = 96.0, 200.0, -3.0, 150.5   # nothing in (0, 96)
        lab[1, 2, :len(B_EDGE_ROW)] = B_EDGE_ROW
        b, y, xx, v = B_OFFSET_PIXEL
        lab[b, y, xx] = v
        x[b, :, y, xx] += 1000.0
        b, y, xx, v = B_SPREAD_PIXEL
        lab[b, y, xx] = v
        x[b, :, y, xx] = torch.rand(D, generator=g) * 120.0 - 60.0
    if name == "c":
        lab[0, 3, 5], lab[1, 0, 0], lab[1, 7, 39], lab[0, 4, 4] = 96.0, 150.0, -1.0, 0.0
    return x, torch.from_numpy(lab)


def named_pixels(name: str, label: torch.Tensor, max_disp: int) -> np.ndarray:
    """[n, 3] (image, y, x) whose every channel's gradient the fixture holds: case b's edge pixels, and up to N_BAND pixels of the
    [max_disp - 1, max_disp) band."""
    out = []
    if name == "b":
        out += [(1, 2, i) for i in range(len(B_EDGE_ROW))] + [B_OFFSET_PIXEL[:3], B_SPREAD_PIXEL[:3]]
    band = torch.nonzero((label >= max_disp - 1) & (label < max_disp)).numpy()
    out += [tuple(int(v) for v in r) for r in band[:N_BAND] if tuple(int(v) for v in r) not in out]
    return np.array(out, dtype=np.int64).reshape(-1, 3)


def sample_index(name: str, shape, named: np.ndarray) -> np.ndarray:
    """Flat indices into the volume: every stride-th element, and every channel of each named pixel."""
    B, D, H, W = shape
    idx = [np.arange(0, B * D * H * W, CASES[name]["stride"], dtype=np.int64)]
    for b, y, x in named:
        idx.append(((b * D + np.arange(D)) * H + y) * W + x)
    return np.unique(np.concatenate(idx))


def restate(x: torch.Tensor, label: torch.Tensor, max_disp: int, idx: np.ndarray):
    """Float64 restatement of the loss at the shipped settings, one image at a time: (loss, gradient at the flat indices idx, max |grad|).
    outer = 0 < d < max_disp, inner = 0 < d < max_disp - 1, p = softmax_c(-|c - d*inner| / 0.5) * inner + 1e-40 (a zero target when no
    pixel of the batch is in outer), L = -(1/N) sum outer * sum_c p_c log_softmax(x)_c, dL/dx = -(outer / N) (p - softmax(x) sum_c p)."""
    B, D, H, W = x.shape
    N = B * H * W
    lab = label.double()
    outer_all = (lab > 0) & (lab < max_disp)
    any_outer = bool(outer_all.any())
    c = torch.arange(D, dtype=torch.float64).view(D, 1, 1)
    total, gmax = 0.0, 0.0
    grad_at = np.zeros(len(idx), dtype=np.float64)
    per = D * H * W
    for b in range(B):
        d = lab[b]
        outer = outer_all[b].double()
        inner = ((d > 0) & (d < max_disp - 1)).double()
        if any_outer:
            p = torch.softmax(-(c - d * inner).abs() / 0.5, dim=0) * inner + 1e-40
        else:
            p = torch.zeros(D, H, W, dtype=torch.float64)
        ls = torch.log_softmax(x[b].double(), dim=0)
        total += float((p * ls * outer).sum())
        grad = -(outer / N) * (p - ls.exp() * p.sum(0, keepdim=True))
        gmax = max(gmax, float(grad.abs().max()))
        sel = (idx >= b * per) & (idx < (b + 1) * per)
        grad_at[sel] = grad.reshape(-1)[torch.from_numpy(idx[sel] - b * per)].numpy()
    return -total / N, grad_at, gmax


def reference(x: torch.Tensor, label: torch.Tensor, max_disp: int):
    """The unmodified reference's (loss, d loss / d x) on the host."""
    from visualDet3D.networks.heads.losses import DisparityLoss
    xr = x.clone().requires_grad_(True)
    loss = DisparityLoss(max_disp).criterion(xr, label.unsqueeze(1), variance=0.5)
    loss.backward()
    return loss.detach(), xr.grad


def run_case(name: str):
    c = CASES[name]
    x, label = inputs(name)
    D = c["D"]
    loss, grad = reference(x, label, D)
    named = named_pixels(name, label, D)
    idx = sample_index(name, x.shape, named)
    loss64, _, _ = restate(x, label, D, idx)
    out = dict(B=c["B"], D=D, H=c["H"], W=c["W"], max_disp=D, seed=c["seed"], x_sha=np.array(sha(x)), label_sha=np.array(sha(label)),
               loss=loss.numpy().astype(np.float32), loss64=np.float64(loss64), grad_idx=idx, grad=grad.reshape(-1)[idx].numpy(),
               grad_max=np.float32(grad.abs().max()), named=named, outer_count=np.int64(((label > 0) & (label < D)).sum()))
    print(f"case {name}: loss {float(loss):.9g} (float64 {loss64:.9g}) outer {int(out['outer_count'])} / {label.numel()}  "
          f"grad max {float(out['grad_max']):.4g}  samples {len(idx)}  named {len(named)}")
    return out


def main():
    import refload
    refload.load_reference()
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    fix = {}
    for name in CASES:
        for k, v in run_case(name).items():
            fix[f"{name}/{k}"] = v
    path = os.path.join(HERE, "disparity_loss.npz")
    np.savez_compressed(path, **fix)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
