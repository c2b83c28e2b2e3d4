"""The tile lists of the anchor head's regression tower (vd3d_reg_tower_tiles) restated in numpy, and the constructed candidate maps both the
CPU and the GPU tests run it on.

For depth d the tower conv must be right at S_d, the pixels within d 3x3 steps (Chebyshev distance d) of a candidate pixel.  Per image the
8 x 16 tiles start at the first row of S_d, and a tile is listed when it holds a pixel of S_d; the list is ordered image, tile row, tile column."""
import numpy as np

TH, TW = 8, 16


def cap(B, H, W):
    return B * (-(-H // TH) + 1) * -(-W // TW)


def dilate(cand, d):
    """[B, H, W] bool -> the pixels within d 3x3 steps of a set pixel, clipped to the image (d steps of a 3x3 max filter)"""
    s = cand.astype(bool).copy()
    B, H, W = s.shape
    for _ in range(d):
        p = np.zeros((B, H + 2, W + 2), dtype=bool)
        p[:, 1:-1, 1:-1] = s
        s = np.zeros_like(s)
        for dy in range(3):
            for dx in range(3):
                s |= p[:, dy:dy + H, dx:dx + W]
    return s


def tiles(cand, d):
    """-> (S_d [B, H, W] bool, list [n, 4] int32 of (b, y0, x0, 0))"""
    s = dilate(cand, d)
    B, H, W = s.shape
    out = []
    for b in range(B):
        ys = np.nonzero(s[b].any(1))[0]
        if len(ys) == 0:
            continue
        for y0 in range(int(ys[0]), H, TH):
            for x0 in range(0, W, TW):
                if s[b, y0:y0 + TH, x0:x0 + TW].any():
                    out.append((b, y0, x0, 0))
    return s, np.array(out, dtype=np.int32).reshape(-1, 4)


def maps():
    """name -> constructed candidate map [B, H, W] uint8"""
    rng = np.random.default_rng(11)
    m = {}
    B, H, W = 3, 24, 80                       # the bench's stride-16 map (384 x 1280), three images
    m["empty"] = np.zeros((B, H, W), np.uint8)
    z = np.zeros((B, H, W), np.uint8)
    z[0, 0, 0] = z[1, 0, W - 1] = z[2, H - 1, 0] = 1
    z[2, H - 1, W - 1] = 1
    m["corners"] = z
    z = np.zeros((B, H, W), np.uint8)
    z[0, 0, :] = 1                             # a band at the top edge, one at the bottom edge, none in image 1
    z[2, H - 2:, 3:50] = 1
    m["edge_bands"] = z
    m["full"] = np.ones((B, H, W), np.uint8)
    m["bench_like"] = (rng.random((B, H, W)) < 0.02).astype(np.uint8) * (np.arange(H)[None, :, None] // 5 == 1)
    m["ragged"] = (rng.random((2, 13, 37)) < 0.03).astype(np.uint8)     # H not a multiple of 8, W not of 16
    m["single_row"] = (rng.random((2, 1, 20)) < 0.2).astype(np.uint8)
    m["dense_random"] = (rng.random((4, 24, 80)) < 0.3).astype(np.uint8)
    return m
