"""ORACLE infrastructure (not product code): cv2.StereoBM_create(192, 25).compute restated in numpy, at the one setting the reference's
disparity precompute uses (scripts/disparity_compute.py): 192 disparities, a 25x25 window, and cv2's defaults for everything else
(XSOBEL prefilter with cap 31, texture threshold 10, uniqueness ratio 15, no speckle filter, no left-right check, minDisparity 0).

Restates cv2's documented behaviour, not the reference; checked bit for bit against cv2 4.13 by tests/test_disparity_gt_cpu.py.

    grey(img)                     cv2.cvtColor(uint8 HWC, COLOR_BGR2GRAY)
    denorm(img, mean, std)        the precompute script's de-normalisation of a float32 HWC network input to uint8
    prefilter(g)                  the XSOBEL prefilter, uint8 values 0..62
    cost_volume(gl, gr)           C[i, y, x] (i = ND-1-d) and the texture sum T[y, x] on the valid region (elsewhere 0)
    stereo_bm(gl, gr)             the int16 disparity map (16 x pixels, -16 = filtered)
    block_max(disp)               skimage.measure.block_reduce(max(disp, 0) as uint16, (4, 4), np.max): zero-padded far edges
"""
import numpy as np

ND = 192
WIN = 25
HW = WIN // 2                 # 12
CAP = 31
TEXTURE = 10
UNIQUENESS = 15
FILTERED = -16
X0 = ND - 1 + HW              # 203: the first column with an output
MIN_H, MIN_W = 26, 216        # the smallest frame with a defined map (cv2 rejects H <= 25; below W = 216 no column is computed)


def grey(img: np.ndarray) -> np.ndarray:
    """COLOR_BGR2GRAY on uint8: channel 0 is weighted as blue."""
    c = img.astype(np.int64)
    return ((c[..., 0] * 3735 + c[..., 1] * 19235 + c[..., 2] * 9798 + 16384) >> 15).astype(np.uint8)


def denorm(img: np.ndarray, mean: np.ndarray, std: np.ndarray) -> np.ndarray:
    """`image * rgb_std + rgb_mean` in float64, clipped to [0, 1], times 255, truncated to uint8."""
    v = img * np.asarray(std, np.float64)
    v = v + np.asarray(mean, np.float64)
    v[v > 1] = 1
    v[v < 0] = 0
    v *= 255
    return np.array(v, dtype=np.uint8)


def prefilter(g: np.ndarray) -> np.ndarray:
    H, W = g.shape
    gi = g.astype(np.int32)
    up = np.concatenate([gi[1:2], gi[:-1]], 0)            # row -1 reads row 1 (reflect-101)
    dn = np.concatenate([gi[1:], gi[H - 2:H - 1]], 0)     # row H reads row H-2
    s = np.zeros((H, W), np.int32)
    dx = lambda a: a[:, 2:] - a[:, :-2]
    s[:, 1:-1] = dx(up) + 2 * dx(gi) + dx(dn)
    p = np.clip(s, -CAP, CAP) + CAP
    p[:, 0] = CAP
    p[:, -1] = CAP
    if H % 2:
        p[-1] = CAP                                        # cv2 filters rows in pairs: an odd last row stays 31
    return p.astype(np.uint8)


def _box(a: np.ndarray) -> np.ndarray:
    """25x25 window sums of a [..., H, W] int32 array, centred; valid where the window fits (elsewhere 0)."""
    c = np.cumsum(np.cumsum(a, -2, dtype=np.int64), -1)
    c = np.pad(c, [(0, 0)] * (a.ndim - 2) + [(1, 0), (1, 0)])
    out = np.zeros(a.shape, np.int64)
    s = c[..., WIN:, WIN:] - c[..., :-WIN, WIN:] - c[..., WIN:, :-WIN] + c[..., :-WIN, :-WIN]
    out[..., HW:a.shape[-2] - HW, HW:a.shape[-1] - HW] = s
    return out


def cost_volume(gl: np.ndarray, gr: np.ndarray):
    """(C [ND, H, W] int32 with C[i] the cost of disparity ND-1-i, T [H, W] int32) from two uint8 grey images.  Only pixels with an
    output (rows 12..H-13, columns 203..W-13) hold values."""
    H, W = gl.shape
    pl, pr = prefilter(gl).astype(np.int32), prefilter(gr).astype(np.int32)
    C = np.zeros((ND, H, W), np.int32)
    for d in range(ND):
        diff = np.zeros((H, W), np.int32)
        diff[:, d:] = np.abs(pl[:, d:] - pr[:, :W - d])
        C[ND - 1 - d] = _box(diff)
    T = _box(np.abs(pl - CAP)).astype(np.int32)
    mask = valid_mask(H, W)
    C[:, ~mask] = 0
    T[~mask] = 0
    return C, T


def valid_mask(H: int, W: int) -> np.ndarray:
    m = np.zeros((H, W), bool)
    m[HW:H - HW, X0:W - HW] = True
    return m


def decide(C: np.ndarray, T: np.ndarray) -> np.ndarray:
    """The decision of every pixel from its cost vector C[:, y, x] and texture T[y, x]; int16."""
    ND_, H, W = C.shape
    mind = np.argmin(C, 0)                                 # first index of the smallest cost: ties go to the larger disparity
    yy, xx = np.mgrid[0:H, 0:W]
    minsad = C[mind, yy, xx].astype(np.int64)
    thresh = minsad + minsad * UNIQUENESS // 100
    j = np.arange(ND_)[:, None, None]
    far = (j < mind[None] - 1) | (j > mind[None] + 1)
    not_unique = np.any(far & (C <= thresh[None]), 0)
    p = C[np.minimum(mind + 1, ND_ - 1), yy, xx].astype(np.int64)
    n = C[np.maximum(mind - 1, 0), yy, xx].astype(np.int64)
    p = np.where(mind == ND_ - 1, C[ND_ - 2, yy, xx], p)   # sad[ND] := sad[ND-2]
    n = np.where(mind == 0, C[1, yy, xx], n)               # sad[-1] := sad[1]
    den = p + n - 2 * minsad + np.abs(p - n)
    num = (p - n) * 256
    q = np.zeros_like(num)
    nz = den != 0
    q[nz] = np.trunc(num[nz] / den[nz]).astype(np.int64)  # C truncating division (|num| < 2^24: exact in float64)
    out = ((ND_ - 1 - mind) * 256 + q + 15) >> 4
    out = np.where((T < TEXTURE) | not_unique, FILTERED, out)
    return out.astype(np.int16)


def stereo_bm(gl: np.ndarray, gr: np.ndarray) -> np.ndarray:
    H, W = gl.shape
    if H < MIN_H or W < MIN_W:
        raise ValueError(f"{H}x{W}: StereoBM(192, 25) needs at least {MIN_H}x{MIN_W}")
    C, T = cost_volume(gl, gr)
    out = decide(C, T)
    out[~valid_mask(H, W)] = FILTERED
    return out


def block_max(disp: np.ndarray) -> np.ndarray:
    """max(disp, 0) as uint16, then the 4x4 block max with the far edges zero-padded: [ceil(H/4), ceil(W/4)]."""
    d = np.maximum(disp.astype(np.int64), 0).astype(np.uint16)
    H, W = d.shape
    Ho, Wo = -(-H // 4), -(-W // 4)
    pad = np.zeros((Ho * 4, Wo * 4), np.uint16)
    pad[:H, :W] = d
    return pad.reshape(Ho, 4, Wo, 4).max((1, 3))
