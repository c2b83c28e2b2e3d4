// cv2.resize INTER_LINEAR geometry shared by the test-time input pipeline (preprocess.cu) and the training augmentation
// (train_augment.cu): the Resize(preserve_aspect_ratio) output size of a CropTop'ed frame and the source index / weight of one
// destination index.  Reference: R/data/pipeline/stereo_augmentator.py:63-134 (Resize), :213-258 (CropTop).
#pragma once
#include <math.h>

namespace vd3d {

// cv2.resize INTER_LINEAR source index / weight of destination index d (resize.cpp: fx = (d + 0.5) * scale - 0.5, clamped at the borders)
__host__ __device__ inline void lin_coord(int d, double scale, int n, int* s0, float* w1) {
    const double fd = (d + 0.5) * scale - 0.5;       // fraction taken in double (what the IPP-backed cv2 builds do; OpenCV's own C++ path
    int s = (int)floor(fd);                           // rounds the coordinate to float32 first, moving the weight by up to 6e-5 at x ~ 1000)
    float f = (float)(fd - (double)s);
    if (s < 0) { f = 0.f; s = 0; }
    if (s >= n - 1) { f = 0.f; s = n - 1; }
    *s0 = s; *w1 = f;
}

// Resize(size) with preserve_aspect_ratio on a frame of Hc x W rows / columns (after CropTop): scale_factor = size[0] / Hc, the resized
// size np.round(Hc * scale_factor) x np.round(W * scale_factor), and cv2's per-axis source step 1 / (dst / src).
struct ResizeGeom {
    int Hr, Wr;
    double scale_y, scale_x;
};

static inline ResizeGeom resize_geom(int Hc, int W, int Ho) {
    ResizeGeom g;
    const double sf = (double)Ho / (double)Hc;
    g.Hr = (int)nearbyint((double)Hc * sf);            // np.round
    g.Wr = (int)nearbyint((double)W * sf);
    g.scale_y = 1.0 / ((double)g.Hr / (double)Hc);     // cv2: inv_scale = dsize / ssize, scale = 1 / inv_scale
    g.scale_x = 1.0 / ((double)g.Wr / (double)W);
    return g;
}

}  // namespace vd3d
