"""Golden vectors for visualdet3d_b200/train_augment.py from the UNMODIFIED reference `Compose` (build_augmentator) of the five shipped
train_augmentation lists (tests/train_augment_cases.py), on seeded uint8 frames of three KITTI sizes with P2 / P3 and six labels.
Seeds are picked so that, over each list's cases, every branch is taken: both mirror outcomes and both contrast orders of
PhotometricDistort (chain 1); all six Shuffle orders, both mirror outcomes and a warp centre near the frame border (chain 2).
Per case: strided samples, sums, the first row and last column of each output image (CHW), P2 / P3, the kept labels after the chain and
the next np.random.rand() after the call.   python tests/golden/make_golden_train_augment.py"""
import os
import sys
from copy import deepcopy

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (os.path.dirname(HERE), ROOT, os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)
import refload  # noqa: E402
import train_augment_cases as cases  # noqa: E402


def edict(x):
    if isinstance(x, dict):
        return refload.EasyDict({k: edict(v) for k, v in x.items()})
    if isinstance(x, list):
        return [edict(v) for v in x]
    return x


class _Obj:
    pass


def branch(name, seed, H, W):
    """The branches the chain takes from `seed` (read off the host module's program; the fixtures pin the module to the reference)."""
    from visualdet3d_b200.train_augment import TrainAugmentation
    aug_list, stereo = cases.LISTS[name]
    np.random.seed(seed)
    img = np.zeros((H, W, 3), np.uint8)
    out = TrainAugmentation(aug_list)(img, img if stereo else None, cases.P2.copy(), cases.P3.copy() if stereo else None, [])
    f = out[0]
    ops = [int(o) for o in f.ops]
    if name in ("monoflex", "km3d"):
        first = [ops.index(c) for c in (1, 2, 3)]                        # brightness, contrast, the HSV saturation Compose
        order = tuple(int(i) for i in np.argsort(first))
        np.random.seed(seed)
        np.random.uniform()
        cw, ch = np.random.randint(128, W - 128), np.random.randint(128, H - 128)
        border = min(cw - 128, W - 129 - cw) < 24 or min(ch - 128, H - 129 - ch) < 8
        return f.mirror, order, border
    return f.mirror, ops.index(2) < ops.index(3)                         # contrast before the HSV round trip


def pick_seeds(name):
    chain2 = name in ("monoflex", "km3d")
    seen_m, seen_o, border, seeds = set(), set(), False, []
    for s in range(1000):
        H, W = cases.SIZES[len(seeds) % 3]
        seed = 1000 * cases.NAMES.index(name) + s
        b = branch(name, seed, H, W)
        if chain2:                                                       # every Shuffle order, both mirrors, one centre near the border
            new = b[0] not in seen_m or b[1] not in seen_o or (b[2] and not border)
            key = b[1]
        else:                                                            # every (mirror, contrast order) pair
            key = (b[0], b[1])
            new = key not in seen_o
        if new:
            seeds.append(seed)
            seen_m.add(b[0])
            seen_o.add(key)
            border = border or (chain2 and b[2])
        if len(seen_o) == (6 if chain2 else 4) and len(seen_m) == 2 and (border or not chain2):
            return seeds
    raise RuntimeError(f"{name}: no seed set covers every branch")


def main():
    refload.load_reference()
    from visualDet3D.data.pipeline import build_augmentator
    from visualDet3D.data.kitti.kittidata import KittiObj
    out = {}
    for name in cases.NAMES:
        aug_list, stereo = cases.LISTS[name]
        compose = build_augmentator(edict(aug_list))
        seeds = pick_seeds(name)
        for ci, seed in enumerate(seeds):
            H, W = cases.SIZES[ci % 3]
            left, right = cases.frame(seed, H, W), cases.frame(seed + 1, H, W)
            objs = cases.labels(seed, H, W, KittiObj)
            np.random.seed(seed)
            if stereo:
                lo, ro, p2, p3, lab = compose(left, right, deepcopy(cases.P2), deepcopy(cases.P3), deepcopy(objs))
                imgs = {"l": lo, "r": ro}
            else:
                lo, p2, lab = compose(left, p2=deepcopy(cases.P2), labels=deepcopy(objs))
                p3 = np.zeros((3, 4))
                imgs = {"l": lo}
            nxt = np.random.rand()
            k = f"{name}_{ci}"
            out[f"{k}_meta"] = np.array([seed, H, W, int(stereo)])
            out[f"{k}_P2"], out[f"{k}_P3"] = p2, p3
            out[f"{k}_labels"] = cases.label_array(lab)
            out[f"{k}_next_rand"] = np.float64(nxt)
            for side, im in imgs.items():
                chw = np.ascontiguousarray(im.transpose(2, 0, 1))                # collate_fn: [H, W, 3] -> [3, H, W]
                st = max(1, chw.size // 2048)
                out[f"{k}_{side}_stride"] = np.int64(st)
                out[f"{k}_{side}_samples"] = chw.reshape(-1)[::st].astype(np.float32)
                out[f"{k}_{side}_sum"] = np.float64(chw.astype(np.float64).sum())
                out[f"{k}_{side}_abssum"] = np.float64(np.abs(chw.astype(np.float64)).sum())
                out[f"{k}_{side}_first_row"] = chw[:, 0, :].astype(np.float32)
                out[f"{k}_{side}_last_col"] = chw[:, :, -1].astype(np.float32)
            print(f"{k}: seed {seed} {H}x{W} -> {lo.shape}, {len(lab)} labels kept, branch {branch(name, seed, H, W)}")
        out[f"{name}_cases"] = np.int64(len(seeds))
    np.savez_compressed(os.path.join(HERE, "train_augment.npz"), **out)


if __name__ == "__main__":
    main()
