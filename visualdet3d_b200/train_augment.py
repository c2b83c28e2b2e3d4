"""Training-time image augmentation on the GPU: the reference's `train_augmentation` chains (R/data/pipeline/stereo_augmentator.py,
built by augmentation_builder.py's Compose) with the image work moved into one CUDA kernel per batch (csrc/train_augment.cu).

`TrainAugmentation(aug_list)` is a drop-in for `build_augmentator(aug_list)` on the five shipped training lists (Stereo3D, Yolo3D /
GroundAwareYolo3D, RetinaNet, MonoFlex, KM3D).  Per call it
  * draws the random parameters with the same `numpy.random` calls, in the same order and with the same arguments, as the reference
    transforms, so the global RNG ends where the reference leaves it;
  * updates P2 / P3 and the labels on the host with the reference's float64 operations in the reference's order (CropTop, Resize,
    RandomWarpAffine, RandomMirror, FilterObject);
  * returns a `DeferredFrame` in place of each image: the untouched uint8 frame plus what the kernel needs to produce the float32 network
    input.  `.shape` is the (Ho, Wo, 3) of the image the reference would have returned.
`DeferredBatch(frames)` stacks a batch's DeferredFrames into one uint8 staging buffer (what the collate_fn of
`plugin.install_train_augmentation_into_reference()` hands the training step); `DeferredBatch.to_device` / `augment_batch(frames, device)`
turn it into the [B, 3, Ho, Wo] float32 batch with one upload and one launch;
`augment_host(frame)` is the host form of the same per-pixel routine (the parity checker)."""
from __future__ import annotations

import ctypes
import math
import re
from typing import List, Sequence

import numpy as np
import torch
from numpy import random

from . import _lib

GEOM_RESIZE, GEOM_WARP_U8, GEOM_WARP_F32 = 0, 1, 2
OP_BRIGHTNESS, OP_CONTRAST, OP_RGB2HSV, OP_SATURATION, OP_HUE, OP_HSV2RGB, OP_EIGEN_NOISE = range(1, 8)
MAX_OPS = 8

# RandomEigenvalueNoise's defaults: the ImageNet RGB PCA (AlexNet's "fancy PCA" lighting noise)
EIG_VAL = np.array([0.2141788, 0.01817699, 0.00341571], dtype=np.float32)
EIG_VEC = np.array([[-0.58752847, -0.69563484, 0.41340352],
                    [-0.5832747, 0.00994535, -0.81221408],
                    [-0.56089297, 0.71832671, 0.41158938]], dtype=np.float32)


def _vp(a: np.ndarray):
    return a.ctypes.data_as(ctypes.c_void_p)


class DeferredFrame:
    """One augmented image, not yet computed: the uint8 HWC frame and the per-image kernel parameters."""
    __slots__ = ("frame", "geom", "crop_top", "affine", "mirror", "ops", "args", "noise", "shape", "mean", "std")

    def __init__(self, frame, geom, crop_top, affine, mirror, ops, args, noise, Ho, Wo, mean, std):
        self.frame = np.ascontiguousarray(frame)
        assert self.frame.dtype == np.uint8 and self.frame.ndim == 3, "uint8 HWC frames"      # describe() refuses other than 3 channels
        self.geom, self.crop_top, self.affine, self.mirror = geom, crop_top, affine, mirror
        self.ops, self.args, self.noise = ops, args, noise
        self.shape = (Ho, Wo, 3)
        self.mean, self.std = np.ascontiguousarray(mean, dtype=np.float32), np.ascontiguousarray(std, dtype=np.float32)

    def params(self):
        """Everything but the frame's bytes: (H, W, C) of the frame and the kernel parameters."""
        return (self.frame.shape, self.geom, self.crop_top, self.affine, self.mirror, self.ops, self.args, self.noise, self.shape[:2])

    def describe(self, src_ptr: int) -> np.ndarray:
        """The packed kernel descriptor of this frame read from `src_ptr` (host or device address of the frame's bytes)."""
        return _describe(src_ptr, *self.params())


def _describe(src_ptr, hwc, geom, crop_top, affine, mirror, ops, args, noise, out_hw, pitch=None) -> np.ndarray:
    """The packed descriptor of an H x W x C frame at `src_ptr` whose rows are `pitch` bytes apart (default W * C: a packed frame)."""
    desc = np.zeros(int(_lib.load().vd3d_train_augment_desc_bytes()), dtype=np.uint8)
    (H, W, C), (Ho, Wo) = hwc, out_hw
    _lib.call("vd3d_train_augment_describe", _vp(desc), src_ptr, H, W, C, W * C if pitch is None else pitch, geom, crop_top, Ho, Wo, _vp(affine),
              mirror, len(ops), _vp(ops), _vp(args), _vp(noise))
    return desc


def augment_host(f: DeferredFrame) -> np.ndarray:
    """DeferredFrame -> float32 [3, Ho, Wo] on the host (the parity checker of `augment_batch`)."""
    Ho, Wo, _ = f.shape
    out = np.empty((3, Ho, Wo), dtype=np.float32)
    desc = f.describe(f.frame.ctypes.data)
    _lib.call("vd3d_train_augment_host", _vp(desc), 3, Ho, Wo, _vp(f.mean), _vp(f.std), _vp(out))
    return out


class DeferredBatch:
    """The images of one collated batch, not yet computed: the uint8 frames copied into one staging buffer, and each frame's kernel
    parameters.  Built where the batch is collated (a DataLoader worker); `to_device` uploads it and runs the kernel once."""

    def __init__(self, frames: Sequence[DeferredFrame]):
        assert len(frames) > 0
        Ho, Wo, _ = frames[0].shape
        mean, std = frames[0].mean, frames[0].std
        for f in frames:
            assert f.shape == (Ho, Wo, 3), "one output size per batch"
            assert np.array_equal(f.mean, mean) and np.array_equal(f.std, std), "one Normalize per batch"
        sizes = [f.frame.nbytes for f in frames]
        self.offsets = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        self.staging = torch.empty(int(self.offsets[-1]), dtype=torch.uint8)
        host = self.staging.numpy()
        for f, o, n in zip(frames, self.offsets, sizes):
            host[o:o + n] = f.frame.reshape(-1)
        self.params = [f.params() for f in frames]          # the frames' bytes are in `staging`
        self.shape, self.mean, self.std = (len(frames), 3, Ho, Wo), mean, std

    def __len__(self):
        return len(self.params)

    def pin_memory(self):
        self.staging = self.staging.pin_memory()
        return self

    def to_device(self, device="cuda") -> torch.Tensor:
        """[B, 3, Ho, Wo] float32 on `device`: one upload of the staging buffer, one kernel."""
        B, _, Ho, Wo = self.shape
        dev = self.staging.to(device, non_blocking=True)
        descs = np.stack([_describe(dev.data_ptr() + int(o), *p) for p, o in zip(self.params, self.offsets)])
        d = torch.from_numpy(descs).to(device, non_blocking=True)
        out = torch.empty(B, 3, Ho, Wo, dtype=torch.float32, device=device)
        _lib.call("vd3d_train_augment", d.data_ptr(), B, 3, Ho, Wo, _vp(self.mean), _vp(self.std), out.data_ptr(),
                  torch.cuda.current_stream().cuda_stream)
        out._vd3d_keepalive = (self.staging, dev, d)     # the buffers and descriptors must outlive the asynchronous copies and kernel
        return out


def augment_batch(frames: Sequence[DeferredFrame], device="cuda") -> torch.Tensor:
    """DeferredFrames (same output size and Normalize; source sizes may differ) -> [B, 3, Ho, Wo] float32 on `device`: one pinned
    staging copy of the uint8 frames, one upload, one kernel."""
    return DeferredBatch(frames).pin_memory().to_device(device)


# ---------------------------------------------------------------------------------------------------------------------------------
# The transforms.  Each step has a `kind` (one letter, checked against the supported chain shapes at construction) and, for the
# photometric ones, `draw(st)`, which makes the reference transform's numpy.random calls and appends its op to the program.


class _State:
    __slots__ = ("h", "w", "p2", "p3", "labels", "ops", "noise", "geom", "crop_top", "affine", "mirror", "swap", "out_hw", "mean", "std")


def _kw(cfg) -> dict:
    kw = cfg.get("keywords", None)
    return dict(kw) if kw else {}


class _Brightness:
    kind, nops = "P", 1

    def __init__(self, distort_prob, delta=32):
        self.p, self.delta = distort_prob, delta

    def draw(self, st):
        if random.rand() <= self.p:
            st.ops.append((OP_BRIGHTNESS, random.uniform(-self.delta, self.delta)))


class _Contrast:
    kind, nops = "P", 1

    def __init__(self, distort_prob, lower=0.5, upper=1.5):
        self.p, self.lower, self.upper = distort_prob, lower, upper

    def draw(self, st):
        if random.rand() <= self.p:
            st.ops.append((OP_CONTRAST, random.uniform(self.lower, self.upper)))


class _Saturation(_Contrast):
    def draw(self, st):
        if random.rand() <= self.p:
            st.ops.append((OP_SATURATION, random.uniform(self.lower, self.upper)))


class _Hue:
    kind, nops = "P", 1

    def __init__(self, distort_prob, delta=18.0):
        self.p, self.delta = distort_prob, delta

    def draw(self, st):
        if random.rand() <= self.p:
            st.ops.append((OP_HUE, random.uniform(-self.delta, self.delta)))


class _ConvertColor:
    kind, nops = "P", 1

    def __init__(self, current="RGB", transform="HSV"):
        if (current, transform) == ("RGB", "HSV"):
            self.op = OP_RGB2HSV
        elif (current, transform) == ("HSV", "RGB"):
            self.op = OP_HSV2RGB
        else:
            raise NotImplementedError(f"ConvertColor({current} -> {transform})")

    def draw(self, st):
        st.ops.append((self.op, 0.0))


class _EigenNoise:
    kind, nops = "P", 1

    def __init__(self, distort_prob=1.0, alphastd=0.1, eigen_value=EIG_VAL, eigen_vector=EIG_VEC):
        self.p, self.alphastd, self.val, self.vec = distort_prob, alphastd, eigen_value, eigen_vector

    def draw(self, st):
        if random.rand() <= self.p:
            alpha = np.random.normal(scale=self.alphastd, size=(3, ))
            st.noise = np.dot(self.vec, self.val * alpha) * 255           # float64, added to the float32 image in float64
            st.ops.append((OP_EIGEN_NOISE, 0.0))


class _PhotometricDistort:
    kind, nops = "P", 6

    def __init__(self, distort_prob=1.0, contrast_lower=0.5, contrast_upper=1.5, saturation_lower=0.5, saturation_upper=1.5, hue_delta=18.0,
                 brightness_delta=32):
        hsv = [_ConvertColor(), _Saturation(distort_prob, saturation_lower, saturation_upper), _Hue(distort_prob, hue_delta),
               _ConvertColor("HSV", "RGB")]
        self.contrast = _Contrast(distort_prob, contrast_lower, contrast_upper)
        self.brightness = _Brightness(distort_prob, brightness_delta)
        self.first, self.last = [self.contrast] + hsv, hsv + [self.contrast]

    def draw(self, st):
        seq = self.first if random.rand() <= 0.5 else self.last           # contrast before or after the HSV round trip
        for t in [self.brightness] + seq:
            t.draw(st)


class _Sequence:
    """Compose (in order) or Shuffle (in np.random.permutation order) of photometric transforms."""
    kind = "P"

    def __init__(self, aug_list, shuffle):
        self.children = [_build(c) for c in aug_list]
        for c in self.children:
            if c.kind != "P":
                raise NotImplementedError(f"{'Shuffle' if shuffle else 'Compose'} of a non-photometric transform ({type(c).__name__})")
        self.shuffle = shuffle
        self.nops = sum(c.nops for c in self.children)

    def draw(self, st):
        order = np.random.permutation(len(self.children)) if self.shuffle else range(len(self.children))
        for i in order:
            self.children[i].draw(st)


class _ConvertToFloat:
    kind = "F"

    def apply(self, st):
        pass


class _CropTop:
    kind = "C"

    def __init__(self, crop_top_index=None, output_height=None):
        if crop_top_index is None:
            raise NotImplementedError("CropTop without crop_top_index")
        self.upper = crop_top_index

    def apply(self, st):
        upper = self.upper
        st.h -= upper
        st.crop_top = upper
        for p in (st.p2, st.p3):
            if p is not None:
                p[1, 2] = p[1, 2] - upper
                p[1, 3] = p[1, 3] - upper * p[2, 3]
        if st.labels is not None and isinstance(st.labels, list):
            for obj in st.labels:
                obj.bbox_b -= upper
                obj.bbox_t -= upper


class _Resize:
    kind = "R"

    def __init__(self, size, preserve_aspect_ratio=True):
        if not preserve_aspect_ratio or len(size) != 2:
            raise NotImplementedError("Resize other than preserve_aspect_ratio to a (height, width) size")
        self.size = size

    def apply(self, st):
        sf = self.size[0] / st.h
        h = int(np.round(st.h * sf))
        st.geom, st.out_hw = GEOM_RESIZE, (h, self.size[1])
        st.h, st.w = h, self.size[1]
        for p in (st.p2, st.p3):
            if p is not None:
                p[0, :] = p[0, :] * sf
                p[1, :] = p[1, :] * sf
        if st.labels and isinstance(st.labels, list):
            for obj in st.labels:
                obj.bbox_l *= sf
                obj.bbox_r *= sf
                obj.bbox_t *= sf
                obj.bbox_b *= sf


class _WarpAffine:
    kind = "W"

    def __init__(self, scale_lower=0.6, scale_upper=1.4, shift_border=128, output_w=1280, output_h=384):
        self.lower, self.upper, self.border, self.ow, self.oh = scale_lower, scale_upper, shift_border, output_w, output_h
        self.geom = GEOM_WARP_U8                     # GEOM_WARP_F32 when ConvertToFloat comes first (set by TrainAugmentation)

    def apply(self, st):
        s_original = max(st.h, st.w)
        scale = s_original * np.random.uniform(self.lower, self.upper)
        center_w = np.random.randint(low=self.border, high=st.w - self.border)
        center_h = np.random.randint(low=self.border, high=st.h - self.border)
        final_scale = max(self.ow, self.oh) / scale
        final_shift_w = self.ow / 2 - center_w * final_scale
        final_shift_h = self.oh / 2 - center_h * final_scale
        st.affine = np.array([[final_scale, 0, final_shift_w], [0, final_scale, final_shift_h]], dtype=np.float32)
        st.geom, st.out_hw = self.geom, (self.oh, self.ow)
        st.h, st.w = self.oh, self.ow
        for p in (st.p2, st.p3):
            if p is not None:
                p[0:2, :] *= final_scale
                p[0, 2] = p[0, 2] + final_shift_w
                p[0, 3] = p[0, 3] + final_shift_w * p[2, 3]
                p[1, 2] = p[1, 2] + final_shift_h
                p[1, 3] = p[1, 3] + final_shift_h * p[2, 3]
        if st.labels and isinstance(st.labels, list):
            for obj in st.labels:
                obj.bbox_l = obj.bbox_l * final_scale + final_shift_w
                obj.bbox_r = obj.bbox_r * final_scale + final_shift_w
                obj.bbox_t = obj.bbox_t * final_scale + final_shift_h
                obj.bbox_b = obj.bbox_b * final_scale + final_shift_h


class _Mirror:
    kind = "M"

    def __init__(self, mirror_prob):
        self.p = mirror_prob

    def apply(self, st):
        if random.rand() <= self.p:
            st.mirror = 1
            st.swap = not st.swap                     # the reference exchanges the flipped left / right images
            width = st.w
            if st.p2 is not None and st.p3 is not None:
                st.p2, st.p3 = st.p3, st.p2
            for p in (st.p2, st.p3):
                if p is not None:
                    p[0, 3] = -p[0, 3]
                    p[0, 2] = width - p[0, 2] - 1
            if st.labels and isinstance(st.labels, list):
                p2 = st.p2
                for obj in st.labels:
                    obj.bbox_l, obj.bbox_r = width - obj.bbox_r - 1, width - obj.bbox_l - 1
                    z = obj.z
                    obj.x = -obj.x
                    ry = obj.ry
                    ry = (-math.pi - ry) if ry < 0 else (math.pi - ry)
                    while ry > math.pi:
                        ry -= math.pi * 2
                    while ry < (-math.pi):
                        ry += math.pi * 2
                    obj.ry = ry
                    obj.alpha = ry - np.arctan2(obj.x + p2[0, 3] / p2[0, 0], z)     # theta2alpha_3d


class _FilterObject:
    kind = "X"

    def apply(self, st):
        if st.labels is not None:
            keep = []
            if isinstance(st.labels, list):
                for obj in st.labels:
                    if not (obj.bbox_b < 0 or obj.bbox_t > st.h or obj.bbox_r < 0 or obj.bbox_l > st.w):
                        keep.append(obj)
            st.labels = keep


class _Normalize:
    kind = "N"

    def __init__(self, mean, stds):
        self.mean = np.ascontiguousarray(np.array(mean, dtype=np.float32))
        self.std = np.ascontiguousarray(np.array(stds, dtype=np.float32))
        if self.mean.shape != (3, ) or self.std.shape != (3, ):
            raise NotImplementedError("Normalize with other than three channel means / stds")

    def apply(self, st):
        st.mean, st.std = self.mean, self.std


_TYPES = {"ConvertToFloat": _ConvertToFloat, "PhotometricDistort": _PhotometricDistort, "RandomBrightness": _Brightness,
          "RandomContrast": _Contrast, "RandomSaturation": _Saturation, "RandomHue": _Hue, "ConvertColor": _ConvertColor,
          "RandomEigenvalueNoise": _EigenNoise, "CropTop": _CropTop, "Resize": _Resize, "RandomWarpAffine": _WarpAffine,
          "RandomMirror": _Mirror, "FilterObject": _FilterObject, "Normalize": _Normalize}
# chain 1: photometric program on the source frame, then CropTop + Resize; chain 2: warp (before or after ConvertToFloat), then the program
_CHAINS = (re.compile(r"FP*C?R[MX]*N"), re.compile(r"(WF|FW)P*[MX]*N"))


def _build(cfg):
    name = cfg["type_name"]
    kw = _kw(cfg)
    if name in ("Compose", "Shuffle"):
        return _Sequence(kw["aug_list"], shuffle=name == "Shuffle")
    if name not in _TYPES:
        raise NotImplementedError(f"train augmentation {name} has no GPU form")
    return _TYPES[name](**kw)


_RANDOM = {"PhotometricDistort", "RandomBrightness", "RandomContrast", "RandomSaturation", "RandomHue", "RandomEigenvalueNoise",
           "RandomWarpAffine", "RandomMirror", "Shuffle"}


def is_training_list(aug_list) -> bool:
    """True when the list draws random parameters (every shipped training list; no test list does)."""
    def names(lst):
        for c in lst:
            yield c["type_name"]
            if c["type_name"] in ("Compose", "Shuffle"):
                yield from names(_kw(c)["aug_list"])
    return any(n in _RANDOM for n in names(aug_list))


def supports(aug_list) -> bool:
    """True when `TrainAugmentation(aug_list)` can be built."""
    try:
        TrainAugmentation(aug_list)
        return True
    except NotImplementedError:
        return False


class TrainAugmentation:
    """Drop-in for the reference's `build_augmentator(train_augmentation)` with the image work deferred to `augment_batch`."""

    def __init__(self, aug_list):
        self.steps = [_build(c) for c in aug_list]
        kinds = "".join(s.kind for s in self.steps)
        if not any(c.fullmatch(kinds) for c in _CHAINS) or kinds.count("M") > 1:
            raise NotImplementedError(f"train augmentation sequence {[c['type_name'] for c in aug_list]} has no GPU form")
        nops = sum(s.nops for s in self.steps if s.kind == "P")
        if nops > MAX_OPS:
            raise NotImplementedError(f"photometric program of up to {nops} ops (at most {MAX_OPS})")
        if kinds.startswith("FW"):
            self.steps[1].geom = GEOM_WARP_F32

    def __call__(self, left_image, right_image=None, p2=None, p3=None, labels=None, image_gt=None, lidar=None):
        if image_gt is not None or lidar is not None:
            raise NotImplementedError("image_gt / lidar have no GPU augmentation")
        st = _State()
        st.h, st.w = left_image.shape[0:2]
        st.p2, st.p3, st.labels = p2, p3, labels
        st.ops, st.noise, st.crop_top, st.affine, st.mirror, st.swap = [], None, 0, None, 0, False
        for s in self.steps:
            if s.kind == "P":
                s.draw(st)
            else:
                s.apply(st)
        ops = np.array([o for o, _ in st.ops], dtype=np.int32)
        args = np.array([a for _, a in st.ops], dtype=np.float32)          # numpy's float32 in-place op rounds its python float once
        noise = np.zeros(3) if st.noise is None else np.ascontiguousarray(st.noise, dtype=np.float64)
        affine = np.zeros((2, 3), dtype=np.float32) if st.affine is None else st.affine
        Ho, Wo = st.out_hw

        def deferred(frame):
            return DeferredFrame(frame, st.geom, st.crop_top, affine, st.mirror, ops, args, noise, Ho, Wo, st.mean, st.std)

        left, right = (right_image, left_image) if st.swap and right_image is not None else (left_image, right_image)
        out = [deferred(left), None if right is None else deferred(right), st.p2, st.p3, st.labels]
        return [item for item in out if item is not None]
