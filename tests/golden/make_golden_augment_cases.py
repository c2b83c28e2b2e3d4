"""Golden outputs for the constructed augmentation cases (tests/augment_cases.py), computed on the CPU with cv2 and numpy in the reference's
order (R/data/pipeline/stereo_augmentator.py):
  chain 1: ConvertToFloat, the photometric program on the whole frame, CropTop, cv2.resize INTER_LINEAR on float32, crop or zero pad on the
           right, RandomMirror, Normalize;
  chain 2: cv2.warpAffine INTER_LINEAR / BORDER_CONSTANT 0 on the uint8 frame (then ConvertToFloat) or on its float32 copy, the program,
           RandomMirror, Normalize;
  the program: numpy's in-place float32 ops and cv2.cvtColor RGB2HSV / HSV2RGB on float32.
`restate()` is that pipeline for explicit parameters.  Before writing, it is checked against the unmodified reference: the seeds of
tests/golden/train_augment.npz are drawn again with the reference transforms' numpy.random calls and run through `restate()`, and every
image must equal what the reference's own Compose returns for the same seed.  Whole images are stored (float32 [3, Ho, Wo] per case).
The zip members carry a fixed timestamp, so a second run writes the same bytes.   python tests/golden/make_golden_augment_cases.py"""
import io
import os
import sys
import zipfile
from copy import deepcopy

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (os.path.dirname(HERE), ROOT, os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)
import augment_cases as ac  # noqa: E402
import train_augment_cases as tac  # noqa: E402

OUT = os.path.join(HERE, "augment_cases.npz")
# RandomEigenvalueNoise's defaults
EIG_VAL = np.array([0.2141788, 0.01817699, 0.00341571], dtype=np.float32)
EIG_VEC = np.array([[-0.58752847, -0.69563484, 0.41340352], [-0.5832747, 0.00994535, -0.81221408],
                    [-0.56089297, 0.71832671, 0.41158938]], dtype=np.float32)


def program(img, ops, args, noise):
    """The photometric program on a float32 HWC image, as the reference transforms apply it."""
    for op, a in zip(ops, args):
        a = float(a)
        if op == ac.OP_BRIGHTNESS:
            img += a
        elif op == ac.OP_CONTRAST:
            img *= a
        elif op == ac.OP_RGB2HSV:
            img = cv2.cvtColor(img, cv2.COLOR_RGB2HSV)
        elif op == ac.OP_SATURATION:
            img[:, :, 1] *= a
        elif op == ac.OP_HUE:
            img[:, :, 0] += a
            img[:, :, 0][img[:, :, 0] > 360.0] -= 360.0
            img[:, :, 0][img[:, :, 0] < 0.0] += 360.0
        elif op == ac.OP_HSV2RGB:
            img = cv2.cvtColor(img, cv2.COLOR_HSV2RGB)
        elif op == ac.OP_EIGEN_NOISE:
            img += np.asarray(noise, np.float64)
        else:
            raise ValueError(op)
    return img


def restate(frame, geom, crop_top, affine, mirror, ops, args, noise, Ho, Wo):
    """uint8 HWC frame -> float32 [3, Ho, Wo] network input."""
    if geom == ac.GEOM_RESIZE:
        img = program(frame.astype(np.float32), ops, args, noise)
        img = img[crop_top:]
        sf = Ho / img.shape[0]
        h, w = int(np.round(img.shape[0] * sf)), int(np.round(img.shape[1] * sf))
        assert h == Ho
        img = cv2.resize(img, (w, h))
        if w > Wo:
            img = img[:, :Wo]
        elif w < Wo:
            img = np.pad(img, [(0, 0), (0, Wo - w), (0, 0)], "constant")
    else:
        src = frame if geom == ac.GEOM_WARP_U8 else frame.astype(np.float32)
        img = cv2.warpAffine(src, affine, (Wo, Ho), flags=cv2.INTER_LINEAR).astype(np.float32)
        img = program(img, ops, args, noise)
    if mirror:
        img = np.ascontiguousarray(img[:, ::-1, :])
    img = img.astype(np.float32)
    img /= 255.0
    img -= ac.MEAN
    img /= ac.STD
    return np.ascontiguousarray(img.transpose(2, 0, 1))


# ---- the check against the reference --------------------------------------------------------------------------------------------------
def draw(name, H, W):
    """The reference transforms' numpy.random calls for one shipped list, in their order -> restate() parameters (without the frame)."""
    rnd = np.random
    ops = []
    if name in ("monoflex", "km3d"):
        scale = max(H, W) * rnd.uniform(0.6, 1.4)
        cw, ch = rnd.randint(low=128, high=W - 128), rnd.randint(low=128, high=H - 128)
        fs = max(1280, 384) / scale
        affine = np.array([[fs, 0, 1280 / 2 - cw * fs], [0, fs, 384 / 2 - ch * fs]], dtype=np.float32)
        for i in rnd.permutation(3):                                      # Shuffle(brightness, contrast, Compose(HSV saturation))
            if i == 0:
                rnd.rand()
                ops.append((ac.OP_BRIGHTNESS, rnd.uniform(-32, 32)))
            elif i == 1:
                rnd.rand()
                ops.append((ac.OP_CONTRAST, rnd.uniform(0.6, 1.4)))
            else:
                rnd.rand()
                ops += [(ac.OP_RGB2HSV, 0.0), (ac.OP_SATURATION, rnd.uniform(0.6, 1.4)), (ac.OP_HSV2RGB, 0.0)]
        noise = np.zeros(3)
        if name == "km3d":
            rnd.rand()
            alpha = rnd.normal(scale=0.1, size=(3, ))
            noise = np.dot(EIG_VEC, EIG_VAL * alpha) * 255
            ops.append((ac.OP_EIGEN_NOISE, 0.0))
        mirror = int(rnd.rand() <= 0.5)
        geom = ac.GEOM_WARP_U8 if name == "monoflex" else ac.GEOM_WARP_F32
        return dict(geom=geom, crop_top=0, affine=affine, mirror=mirror, ops=[o for o, _ in ops], args=[a for _, a in ops], noise=noise,
                    Ho=384, Wo=1280)
    first = rnd.rand() <= 0.5                                             # PhotometricDistort: contrast before the HSV round trip
    rnd.rand()
    ops.append((ac.OP_BRIGHTNESS, rnd.uniform(-32, 32)))
    if first:
        rnd.rand()
        ops.append((ac.OP_CONTRAST, rnd.uniform(0.5, 1.5)))
    ops.append((ac.OP_RGB2HSV, 0.0))
    rnd.rand()
    ops.append((ac.OP_SATURATION, rnd.uniform(0.5, 1.5)))
    rnd.rand()
    ops.append((ac.OP_HUE, rnd.uniform(-18.0, 18.0)))
    ops.append((ac.OP_HSV2RGB, 0.0))
    if not first:
        rnd.rand()
        ops.append((ac.OP_CONTRAST, rnd.uniform(0.5, 1.5)))
    mirror = int(rnd.rand() <= 0.5)
    return dict(geom=ac.GEOM_RESIZE, crop_top=100, affine=None, mirror=mirror, ops=[o for o, _ in ops], args=[a for _, a in ops],
                noise=np.zeros(3), Ho=288, Wo=1280)


def check_against_reference():
    import refload
    refload.load_reference()
    from visualDet3D.data.pipeline import build_augmentator
    fx = np.load(os.path.join(HERE, "train_augment.npz"))
    worst, n = 0.0, 0
    for name in tac.NAMES:
        aug_list, stereo = tac.LISTS[name]
        compose = build_augmentator(_edict(aug_list))
        for ci in range(int(fx[f"{name}_cases"])):
            seed, H, W, _ = [int(v) for v in fx[f"{name}_{ci}_meta"]]
            left, right = tac.frame(seed, H, W), tac.frame(seed + 1, H, W)
            np.random.seed(seed)
            if stereo:
                ref = compose(left, right, deepcopy(tac.P2), deepcopy(tac.P3), [])[:2]
            else:
                ref = compose(left, p2=deepcopy(tac.P2), labels=[])[:1]
            after = np.random.rand()
            np.random.seed(seed)
            prm = draw(name, H, W)
            assert np.random.rand() == after, (name, seed, "the restated draws leave the RNG elsewhere")
            srcs = [left, right][:len(ref)]
            if stereo and prm["mirror"]:                                  # the reference's mirror exchanges the cameras
                srcs = srcs[::-1]
            for src, r in zip(srcs, ref):
                got = restate(src, **prm)
                want = np.ascontiguousarray(r.transpose(2, 0, 1))
                d = float(np.abs(got - want).max())
                worst, n = max(worst, d), n + 1
                assert d == 0.0, (name, seed, d)
    print(f"restatement vs the reference Compose: {n} images over the train_augment.npz seeds, max |diff| {worst:.1e}")


def _edict(x):
    import refload
    if isinstance(x, dict):
        return refload.EasyDict({k: _edict(v) for k, v in x.items()})
    if isinstance(x, list):
        return [_edict(v) for v in x]
    return x


def write_npz(path, arrays):
    """np.savez_compressed with a fixed member timestamp: the same arrays give the same bytes."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asarray(arrays[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


def main():
    check_against_reference()
    out = {}
    for c in ac.CASES:
        out[c["id"]] = restate(c["frame"], c["geom"], c["crop_top"], c["affine"], c["mirror"], c["ops"], c["args"], c["noise"], c["Ho"], c["Wo"])
    write_npz(OUT, out)
    print(f"{len(out)} cases -> {OUT} ({os.path.getsize(OUT) / 1e6:.2f} MB), cv2 {cv2.__version__}")


if __name__ == "__main__":
    main()
