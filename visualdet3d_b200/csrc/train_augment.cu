// Image input pipelines: uint8 HWC frame -> photometric program / geometry / mirror / Normalize -> CHW float32.  Reference:
// R/data/pipeline/stereo_augmentator.py (ConvertToFloat :29-36, Normalize :39-60, Resize :63-134, RandomSaturation :188-211, CropTop
// :213-258, RandomMirror :373-437, RandomWarpAffine :439-500, RandomHue :502-525, ConvertColor :528-554, RandomContrast :557-578,
// RandomBrightness :580-598, RandomEigenvalueNoise :600-628, PhotometricDistort :630-668).
//
// Two geometries:
//   chain 1 (Stereo3D / Yolo3D / RetinaNet): the photometric program runs on SOURCE pixels, then CropTop + Resize (cv2 INTER_LINEAR on
//     float32, aspect preserved, cropped / zero padded on the right to Wo);
//   chain 2 (MonoFlex / KM3D): cv2.warpAffine (INTER_LINEAR, BORDER_CONSTANT 0, cv2's fixed-point source coordinates) on the uint8 frame
//     (MonoFlex: the warp runs before ConvertToFloat) or on its float32 copy (KM3D), then the photometric program on the warped values.
// Then the mirror (a flip of the finished Wo-wide image: the zero pad of chain 1 ends up on the left) and Normalize.
// Geometry 0 (AUG_RESIZE) with no ops and no mirror is the test-time pipeline (the reference's `test_augmentation`: ConvertToFloat,
// CropTop, Resize, Normalize); the other combinations are the image half of its `train_augmentation` chains.
//
// One routine per output pixel (aug_pixel) is shared by the host entry (vd3d_train_augment_host: the parity checker) and the CUDA kernel
// (one launch per batch, frames of different sizes and both cameras of a stereo batch in one grid).  The kernel stages the distorted
// source rows a tile needs in shared memory, so a chain-1 source pixel is read and distorted once per tile instead of once per bilinear tap.
// Built with -fmad=false: every product and sum rounds separately, like numpy's float32 in-place ops and cv2's scalar loops.
#include "common.cuh"
#include <float.h>
#include <string.h>
#include <math.h>

namespace vd3d {

enum { AUG_RESIZE = 0, AUG_WARP_U8 = 1, AUG_WARP_F32 = 2 };
// The photometric program: brightness (+= delta), contrast (*= alpha), cv2 RGB->HSV, saturation (S *= ratio), hue (H += shift with the
// > 360 / < 0 wrap), cv2 HSV->RGB, eigenvalue noise (+= a float64 per-channel vector).  No clamping: the reference does none.
enum { OP_BRIGHTNESS = 1, OP_CONTRAST = 2, OP_RGB2HSV = 3, OP_SATURATION = 4, OP_HUE = 5, OP_HSV2RGB = 6, OP_EIGEN_NOISE = 7 };
constexpr int AUG_MAX_OPS = 8;

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

struct AugImage {
    const unsigned char* src;   // [H][pitch] bytes, 3 interleaved channels (HWC)
    int H, W, pitch;            // original frame
    int Ho, Wo;                 // network input
    int geom;                   // AUG_RESIZE / AUG_WARP_U8 / AUG_WARP_F32
    int crop_top, Hr, Wr;       // AUG_RESIZE: rows removed at the top, size after the resize (before the crop / pad to Wo)
    double scale_y, scale_x;    // AUG_RESIZE: cv2's 1 / (dst / src) per axis
    double m[6];                // AUG_WARP_*: cv2's inverse map (destination -> source) of the forward 2x3 matrix
    int mirror;                 // flip the finished image horizontally
    int nops;
    int op[AUG_MAX_OPS];
    float arg[AUG_MAX_OPS];     // the float32 the numpy in-place op rounds its python float to
    double noise[3];            // OP_EIGEN_NOISE: the float64 vector, added in float64 and rounded once
};

struct AugParams {
    int Ho, Wo;
    float mean[3], stdv[3];
};

// Kernel tile: AUG_TX output columns x AUG_RY output rows.  describe() holds the resize's source step to <= AUG_MAX_SCALE per axis, which
// bounds the source window a tile reads to the shared-memory stage.
constexpr int AUG_TX = 128, AUG_RY = 4;
constexpr int AUG_MAX_SCALE = 2;
constexpr int AUG_STAGE_ROWS = (AUG_RY - 1) * AUG_MAX_SCALE + 3, AUG_STAGE_COLS = (AUG_TX - 1) * AUG_MAX_SCALE + 3;

__host__ __device__ inline int round_half_even(double v) {    // cv2 saturate_cast<int>(double) = cvRound
#ifdef __CUDA_ARCH__
    return __double2int_rn(v);
#else
    return (int)nearbyint(v);
#endif
}

// cv2 color.cpp RGB2HSV_f / HSV2RGB_f scalar formulas on float32 (hrange 360): c0 = R / H, c1 = G / S, c2 = B / V.
__host__ __device__ inline void rgb_to_hsv(float* c) {
    const float r = c[0], g = c[1], b = c[2];
    float v = r, vmin = r;
    if (v < g) v = g;
    if (v < b) v = b;
    if (vmin > g) vmin = g;
    if (vmin > b) vmin = b;
    float diff = v - vmin;
    const float s = diff / (fabsf(v) + FLT_EPSILON);
    diff = 60.f / (diff + FLT_EPSILON);
    float h;
    if (v == r) h = (g - b) * diff;
    else if (v == g) h = (b - r) * diff + 120.f;
    else h = (r - g) * diff + 240.f;
    if (h < 0.f) h = h + 360.f;
    c[0] = h; c[1] = s; c[2] = v;
}

__host__ __device__ inline void hsv_to_rgb(float* c) {
    float h = c[0];
    const float s = c[1], v = c[2];
    float r, g, b;
    if (s == 0.f) {
        r = g = b = v;
    } else {
        const float hscale = 6.f / 360.f;
        h = h * hscale;
        h = fmodf(h, 6.f);
        if (h < 0.f) h = h + 6.f;
        int sector = (int)floorf(h);
        h = h - (float)sector;
        if ((unsigned)sector >= 6u) { sector = 0; h = 0.f; }
        const float t0 = v, t1 = v * (1.f - s), t2 = v * (1.f - s * h), t3 = v * (1.f - s * (1.f - h));
        // cv2's sector_data {{1,3,0}, {1,0,2}, {3,0,1}, {0,2,1}, {0,1,3}, {2,1,0}}: the (b, g, r) table index of each sector, two bits
        // per sector (kept in registers, not an indexed local array)
        const unsigned sb = 0x835u, sg = 0x583u, sr = 0x358u;
        auto tab = [&](unsigned packed) {
            const unsigned i = (packed >> (2 * sector)) & 3u;
            return i == 0 ? t0 : i == 1 ? t1 : i == 2 ? t2 : t3;
        };
        b = tab(sb); g = tab(sg); r = tab(sr);
    }
    c[0] = r; c[1] = g; c[2] = b;
}

__host__ __device__ inline void apply_ops(const AugImage& im, float* c) {
    for (int i = 0; i < im.nops; ++i) {
        const float t = im.arg[i];
        switch (im.op[i]) {
        case OP_BRIGHTNESS: c[0] = c[0] + t; c[1] = c[1] + t; c[2] = c[2] + t; break;
        case OP_CONTRAST: c[0] = c[0] * t; c[1] = c[1] * t; c[2] = c[2] * t; break;
        case OP_RGB2HSV: rgb_to_hsv(c); break;
        case OP_SATURATION: c[1] = c[1] * t; break;
        case OP_HUE:                                  // numpy: two masked in-place ops, the second sees the first's result
            c[0] = c[0] + t;
            if (c[0] > 360.f) c[0] = c[0] - 360.f;
            if (c[0] < 0.f) c[0] = c[0] + 360.f;
            break;
        case OP_HSV2RGB: hsv_to_rgb(c); break;
        case OP_EIGEN_NOISE:                          // float32 image += float64 vector: the ufunc adds in float64, then casts back
            for (int k = 0; k < 3; ++k) c[k] = (float)((double)c[k] + im.noise[k]);
            break;
        }
    }
}

// The source pixel (row, col) of the cropped frame after the photometric program: evaluated on the fly (host form) ...
struct DirectFetch {
    const AugImage* im;
    __host__ __device__ void operator()(int row, int col, float* c) const {
        const unsigned char* p = im->src + (size_t)(row + im->crop_top) * im->pitch + (size_t)col * 3;
        c[0] = (float)p[0]; c[1] = (float)p[1]; c[2] = (float)p[2];
        apply_ops(*im, c);
    }
};

// ... or read from the tile's shared-memory stage (kernel)
struct StageFetch {
    const float* stage;
    int row0, col0, cols;
    __device__ void operator()(int row, int col, float* c) const {
        const float* q = stage + ((row - row0) * cols + (col - col0)) * 3;
        c[0] = q[0]; c[1] = q[1]; c[2] = q[2];
    }
};

__host__ __device__ inline float warp_tap(const AugImage& im, int sy, int sx, int k) {
    return (sy >= 0 && sy < im.H && sx >= 0 && sx < im.W) ? (float)im.src[(size_t)sy * im.pitch + (size_t)sx * 3 + k] : 0.f;
}

// One output pixel (y, x) of the Wo-wide network input, all three channels, normalised.
template <class Fetch>
__host__ __device__ inline void aug_pixel(const AugImage& im, const AugParams& p, int y, int x, const Fetch& fetch, float* v) {
    const int u = im.mirror ? p.Wo - 1 - x : x;       // column of the un-mirrored image
    v[0] = v[1] = v[2] = 0.f;
    if (im.geom == AUG_RESIZE) {
        if (u < im.Wr) {                              // else: the zero pad on the right (before Normalize)
            const int Hc = im.H - im.crop_top;
            int sy, sx; float fy, fx;
            lin_coord(y, im.scale_y, Hc, &sy, &fy);
            lin_coord(u, im.scale_x, im.W, &sx, &fx);
            const int sy1 = sy + 1 < Hc ? sy + 1 : sy, sx1 = sx + 1 < im.W ? sx + 1 : sx;
            float t00[3], t01[3], t10[3], t11[3];
            fetch(sy, sx, t00); fetch(sy, sx1, t01); fetch(sy1, sx, t10); fetch(sy1, sx1, t11);
            const float a0 = 1.f - fx, a1 = fx, b0 = 1.f - fy, b1 = fy;
            for (int k = 0; k < 3; ++k) {
                const float h0 = t00[k] * a0 + t01[k] * a1;       // horizontal pass of the two source rows
                const float h1 = t10[k] * a0 + t11[k] * a1;
                v[k] = h0 * b0 + h1 * b1;                           // vertical pass
            }
        }
    } else {
        // cv2 warpAffine (imgwarp.cpp WarpAffineInvoker, AB_BITS 10, INTER_BITS 5): per-row and per-column offsets rounded to 1/1024 of a
        // pixel, summed, shifted down to 1/32: the integer source pixel and a 5-bit fraction per axis.
        const int X0 = round_half_even((im.m[1] * y + im.m[2]) * 1024) + 16;
        const int Y0 = round_half_even((im.m[4] * y + im.m[5]) * 1024) + 16;
        const int X = (X0 + round_half_even(im.m[0] * u * 1024)) >> 5;
        const int Y = (Y0 + round_half_even(im.m[3] * u * 1024)) >> 5;
        const int sx = X >> 5, sy = Y >> 5, fx = X & 31, fy = Y & 31;
        if (im.geom == AUG_WARP_U8) {                 // remapBilinear on 8u: 15-bit weights (products of the 1/32 steps), rounded back to uint8
            const int w00 = (32 - fy) * (32 - fx), w01 = (32 - fy) * fx, w10 = fy * (32 - fx), w11 = fy * fx;
            for (int k = 0; k < 3; ++k) {
                const int s = (int)warp_tap(im, sy, sx, k) * w00 + (int)warp_tap(im, sy, sx + 1, k) * w01 +
                              (int)warp_tap(im, sy + 1, sx, k) * w10 + (int)warp_tap(im, sy + 1, sx + 1, k) * w11;
                v[k] = (float)((s + 512) >> 10);
            }
        } else {                                      // remapBilinear on 32f: float weights, summed left to right
            const float wx = (float)fx * (1.f / 32.f), wy = (float)fy * (1.f / 32.f);
            const float w00 = (1.f - wy) * (1.f - wx), w01 = (1.f - wy) * wx, w10 = wy * (1.f - wx), w11 = wy * wx;
            for (int k = 0; k < 3; ++k)
                v[k] = warp_tap(im, sy, sx, k) * w00 + warp_tap(im, sy, sx + 1, k) * w01 + warp_tap(im, sy + 1, sx, k) * w10 +
                       warp_tap(im, sy + 1, sx + 1, k) * w11;
        }
        apply_ops(im, v);
    }
    for (int k = 0; k < 3; ++k) {                     // Normalize: /= 255, -= mean, /= std, in float32 like the numpy in-place ops
        float t = v[k] / 255.0f;
        t = t - p.mean[k];
        v[k] = t / p.stdv[k];
    }
}

__global__ void __launch_bounds__(AUG_TX) train_augment_kernel(const AugImage* __restrict__ descs, AugParams p, float* __restrict__ out) {
    __shared__ AugImage im;
    __shared__ float stage[AUG_STAGE_ROWS * AUG_STAGE_COLS * 3];
    static_assert(sizeof(AugImage) % 4 == 0, "descriptor copied as words");
    const int tid = threadIdx.x, b = blockIdx.z;
    for (int i = tid; i < (int)(sizeof(AugImage) / 4); i += AUG_TX) ((int*)&im)[i] = ((const int*)(descs + b))[i];
    __syncthreads();
    const int x0 = blockIdx.x * AUG_TX, y0 = blockIdx.y * AUG_RY;
    const int x1 = min(x0 + AUG_TX, p.Wo) - 1, y1 = min(y0 + AUG_RY, p.Ho) - 1;
    StageFetch sf{stage, 0, 0, 0};
    if (im.geom == AUG_RESIZE) {
        // the un-mirrored columns of this tile that the resize covers, and the source window their bilinear taps read
        int ul = im.mirror ? p.Wo - 1 - x1 : x0, uh = im.mirror ? p.Wo - 1 - x0 : x1;
        uh = min(uh, im.Wr - 1);
        if (ul <= uh) {                               // block-uniform: a tile wholly in the pad stages nothing
            const int Hc = im.H - im.crop_top;
            int r0, r1, c0, c1; float f;
            lin_coord(y0, im.scale_y, Hc, &r0, &f);
            lin_coord(y1, im.scale_y, Hc, &r1, &f);
            lin_coord(ul, im.scale_x, im.W, &c0, &f);
            lin_coord(uh, im.scale_x, im.W, &c1, &f);
            r1 = min(r1 + 1, Hc - 1);
            c1 = min(c1 + 1, im.W - 1);
            const int rows = r1 - r0 + 1, cols = c1 - c0 + 1;
            const DirectFetch df{&im};
            for (int i = tid; i < rows * cols; i += AUG_TX) {
                const int r = i / cols, c = i - r * cols;
                df(r0 + r, c0 + c, stage + i * 3);
            }
            sf = StageFetch{stage, r0, c0, cols};
        }
        __syncthreads();
    }
    const int x = x0 + tid;
    if (x > x1) return;
    const size_t plane = (size_t)p.Ho * p.Wo;
    float* o = out + (size_t)b * 3 * plane + x;
    for (int y = y0; y <= y1; ++y) {
        float v[3];
        aug_pixel(im, p, y, x, sf, v);
        for (int k = 0; k < 3; ++k) o[k * plane + (size_t)y * p.Wo] = v[k];
    }
}

static int set_params(AugParams* p, int C, int Ho, int Wo, const float* mean, const float* stdv) {
    VD3D_REQUIRE(C == 3 && Ho > 0 && Wo > 0 && mean && stdv, "train_augment: bad arguments (C %d, Ho %d, Wo %d)", C, Ho, Wo);
    p->Ho = Ho; p->Wo = Wo;
    for (int c = 0; c < 3; ++c) { p->mean[c] = mean[c]; p->stdv[c] = stdv[c]; }
    return VD3D_OK;
}

}  // namespace vd3d

using namespace vd3d;

extern "C" int vd3d_train_augment_desc_bytes(void) { return (int)sizeof(AugImage); }

extern "C" int vd3d_train_augment_describe(void* desc, const unsigned char* src, int H, int W, int C, int pitch, int geom, int crop_top,
                                           int Ho, int Wo, const float* affine, int mirror, int nops, const int* ops, const float* args,
                                           const double* noise) {
    VD3D_REQUIRE(desc && src && H > 0 && W > 0 && C == 3 && pitch >= W * C && Ho > 0 && Wo > 0 && (mirror == 0 || mirror == 1),
                 "train_augment_describe: bad arguments");
    VD3D_REQUIRE(nops >= 0 && nops <= AUG_MAX_OPS && (nops == 0 || (ops && args)), "train_augment_describe: bad photometric program (%d ops)", nops);
    AugImage im;
    memset(&im, 0, sizeof(im));
    im.src = src; im.H = H; im.W = W; im.pitch = pitch; im.Ho = Ho; im.Wo = Wo; im.geom = geom; im.mirror = mirror; im.nops = nops;
    for (int i = 0; i < nops; ++i) {
        VD3D_REQUIRE(ops[i] >= OP_BRIGHTNESS && ops[i] <= OP_EIGEN_NOISE, "train_augment_describe: unknown op code %d", ops[i]);
        VD3D_REQUIRE(ops[i] != OP_EIGEN_NOISE || noise, "train_augment_describe: eigenvalue noise without its vector");
        im.op[i] = ops[i]; im.arg[i] = args[i];
    }
    if (noise)
        for (int k = 0; k < 3; ++k) im.noise[k] = noise[k];
    if (geom == AUG_RESIZE) {
        VD3D_REQUIRE(crop_top >= 0 && crop_top < H, "train_augment_describe: crop_top %d outside a %d-row frame", crop_top, H);
        const ResizeGeom g = resize_geom(H - crop_top, W, Ho);
        VD3D_REQUIRE(g.Hr == Ho, "train_augment_describe: rounded resized height %d != network height %d", g.Hr, Ho);
        VD3D_REQUIRE(g.scale_y <= AUG_MAX_SCALE && g.scale_x <= AUG_MAX_SCALE,
                     "train_augment_describe: resize shrinks by more than %dx (%.3f, %.3f)", AUG_MAX_SCALE, g.scale_y, g.scale_x);
        im.crop_top = crop_top; im.Hr = g.Hr; im.Wr = g.Wr; im.scale_y = g.scale_y; im.scale_x = g.scale_x;
    } else if (geom == AUG_WARP_U8 || geom == AUG_WARP_F32) {
        VD3D_REQUIRE(affine, "train_augment_describe: warp without its matrix");
        double* M = im.m;                             // cv2 warpAffine: the float32 matrix in double, inverted unless WARP_INVERSE_MAP
        for (int i = 0; i < 6; ++i) M[i] = (double)affine[i];
        double D = M[0] * M[4] - M[1] * M[3];
        VD3D_REQUIRE(D != 0.0 && isfinite(D), "train_augment_describe: singular warp matrix");
        D = 1. / D;
        const double A11 = M[4] * D, A22 = M[0] * D;
        M[0] = A11; M[1] *= -D;
        M[3] *= -D; M[4] = A22;
        const double b1 = -M[0] * M[2] - M[1] * M[5];
        const double b2 = -M[3] * M[2] - M[4] * M[5];
        M[2] = b1; M[5] = b2;
    } else {
        VD3D_REQUIRE(false, "train_augment_describe: unknown geometry %d", geom);
    }
    memcpy(desc, &im, sizeof(im));
    return VD3D_OK;
}

extern "C" int vd3d_train_augment_host(const void* desc, int C, int Ho, int Wo, const float* mean, const float* stdv, float* out) {
    VD3D_REQUIRE(desc && out, "train_augment_host: null argument");
    AugParams p;
    int rc = set_params(&p, C, Ho, Wo, mean, stdv);
    if (rc) return rc;
    AugImage im;
    memcpy(&im, desc, sizeof(im));
    VD3D_REQUIRE(im.Ho == Ho && im.Wo == Wo, "train_augment_host: descriptor made for %dx%d, output %dx%d", im.Ho, im.Wo, Ho, Wo);
    const DirectFetch df{&im};
    const size_t plane = (size_t)Ho * Wo;
    for (int y = 0; y < Ho; ++y)
        for (int x = 0; x < Wo; ++x) {
            float v[3];
            aug_pixel(im, p, y, x, df, v);
            for (int k = 0; k < 3; ++k) out[k * plane + (size_t)y * Wo + x] = v[k];
        }
    return VD3D_OK;
}

// Batched device form: `descs_dev` is a DEVICE array of n records of vd3d_train_augment_desc_bytes() bytes, each built by
// vd3d_train_augment_describe with `src` a device pointer and the same Ho / Wo; out = [n][3][Ho][Wo] float32.
extern "C" int vd3d_train_augment(const void* descs_dev, int n, int C, int Ho, int Wo, const float* mean, const float* stdv, float* out, void* stream) {
    VD3D_REQUIRE(descs_dev && out && n > 0 && n <= 65535, "train_augment: bad arguments");
    AugParams p;
    int rc = set_params(&p, C, Ho, Wo, mean, stdv);
    if (rc) return rc;
    dim3 grid(cdiv(Wo, AUG_TX), cdiv(Ho, AUG_RY), n);
    train_augment_kernel<<<grid, AUG_TX, 0, (cudaStream_t)stream>>>((const AugImage*)descs_dev, p, out);
    VD3D_CHECK_LAUNCH("train_augment");
    return VD3D_OK;
}
