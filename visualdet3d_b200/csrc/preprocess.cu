// Input pipeline of the test-time augmentation (SURVEY.md 8(f) rank 3): uint8 HWC frame -> ConvertToFloat -> CropTop -> Resize
// (cv2.resize, INTER_LINEAR on float32, aspect preserved, then cropped / zero-padded on the right to the network width) -> Normalize
// -> CHW float32.  Reference: R/data/pipeline/stereo_augmentator.py:29-134 (ConvertToFloat, Normalize, Resize), :213-258 (CropTop).
// One routine per output value, shared by the host entry (vd3d_preprocess_host: parity against the reference's cv2 / numpy pipeline on
// the CPU) and the CUDA kernel (vd3d_preprocess: one thread per output pixel, frames of different sizes in one batch).
#include "common.cuh"
#include "resize_common.cuh"
#include <math.h>

namespace vd3d {

struct PreImage {
    const unsigned char* src;   // [H][pitch] bytes, C interleaved channels (HWC)
    int H, W, pitch;            // original frame
    int crop_top;               // rows removed at the top (CropTop)
    int Hr, Wr;                 // size after the resize (before the crop / pad to the network width)
    double scale_y, scale_x;    // cv2: 1 / (dst / src) per axis
};

struct PreParams {
    int C, Ho, Wo;              // output [C][Ho][Wo] per image (Ho == Hr)
    float mean[4], stdv[4];
};

__host__ __device__ inline float pre_value(const PreImage& im, const PreParams& p, int c, int y, int x) {
    float v = 0.f;                                       // zero padding on the right happens BEFORE Normalize
    if (x < im.Wr) {
        const int Hc = im.H - im.crop_top;               // cropped height
        int sy, sx; float fy, fx;
        lin_coord(y, im.scale_y, Hc, &sy, &fy);
        lin_coord(x, im.scale_x, im.W, &sx, &fx);
        const int sy1 = sy + 1 < Hc ? sy + 1 : sy, sx1 = sx + 1 < im.W ? sx + 1 : sx;
        const unsigned char* r0 = im.src + (size_t)(sy + im.crop_top) * im.pitch;
        const unsigned char* r1 = im.src + (size_t)(sy1 + im.crop_top) * im.pitch;
        const float a0 = 1.f - fx, a1 = fx, b0 = 1.f - fy, b1 = fy;
        const float h0 = (float)r0[sx * p.C + c] * a0 + (float)r0[sx1 * p.C + c] * a1;     // horizontal pass of the two source rows
        const float h1 = (float)r1[sx * p.C + c] * a0 + (float)r1[sx1 * p.C + c] * a1;
        v = h0 * b0 + h1 * b1;                                                              // vertical pass
    }
    v = v / 255.0f;                                      // Normalize: /= 255, -= mean, /= std, in float32 like the numpy in-place ops
    v = v - p.mean[c];
    v = v / p.stdv[c];
    return v;
}

__global__ void preprocess_kernel(const PreImage* __restrict__ imgs, PreParams p, float* __restrict__ out) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, b = blockIdx.z;
    if (x >= p.Wo) return;
    const PreImage im = imgs[b];
    for (int c = 0; c < p.C; ++c) out[(((size_t)b * p.C + c) * p.Ho + y) * p.Wo + x] = pre_value(im, p, c, y, x);
}

static int fill(PreImage* im, PreParams* p, const unsigned char* src, int H, int W, int C, int pitch, int crop_top, int Ho, int Wo,
                const float* mean, const float* stdv) {
    VD3D_REQUIRE(src && H > 0 && W > 0 && C >= 1 && C <= 4 && pitch >= W * C && crop_top >= 0 && crop_top < H && Ho > 0 && Wo > 0 && mean && stdv,
                 "preprocess: bad arguments");
    const ResizeGeom g = resize_geom(H - crop_top, W, Ho);
    im->src = src; im->H = H; im->W = W; im->pitch = pitch; im->crop_top = crop_top;
    im->Hr = g.Hr; im->Wr = g.Wr;
    VD3D_REQUIRE(im->Hr == Ho, "preprocess: rounded resized height %d != network height %d", im->Hr, Ho);
    im->scale_y = g.scale_y; im->scale_x = g.scale_x;
    p->C = C; p->Ho = Ho; p->Wo = Wo;
    for (int c = 0; c < C; ++c) { p->mean[c] = mean[c]; p->stdv[c] = stdv[c]; }
    return VD3D_OK;
}

}  // namespace vd3d

using namespace vd3d;

extern "C" int vd3d_preprocess_host(const unsigned char* src, int H, int W, int C, int pitch, int crop_top, int Ho, int Wo,
                                    const float* mean, const float* stdv, float* out) {
    VD3D_REQUIRE(out, "preprocess_host: null output");
    PreImage im; PreParams p;
    int rc = fill(&im, &p, src, H, W, C, pitch, crop_top, Ho, Wo, mean, stdv);
    if (rc) return rc;
    for (int c = 0; c < C; ++c)
        for (int y = 0; y < Ho; ++y)
            for (int x = 0; x < Wo; ++x) out[((size_t)c * Ho + y) * Wo + x] = pre_value(im, p, c, y, x);
    return VD3D_OK;
}

// Batched device form.  `descs` is a DEVICE array of B PreImage records built by vd3d_preprocess_describe on the host (one per frame,
// `src` a device pointer to the uploaded uint8 frame); out = [B][C][Ho][Wo] float32, what the detectors take.
extern "C" int vd3d_preprocess_desc_bytes(void) { return (int)sizeof(PreImage); }

extern "C" int vd3d_preprocess_describe(void* desc_host, const unsigned char* src_dev, int H, int W, int C, int pitch, int crop_top, int Ho, int Wo) {
    VD3D_REQUIRE(desc_host, "preprocess_describe: null descriptor");
    PreParams p;
    const float one[4] = {1.f, 1.f, 1.f, 1.f};
    return fill((PreImage*)desc_host, &p, src_dev, H, W, C, pitch, crop_top, Ho, Wo, one, one);
}

extern "C" int vd3d_preprocess(const void* descs_dev, int B, int C, int Ho, int Wo, const float* mean, const float* stdv, float* out, void* stream) {
    VD3D_REQUIRE(descs_dev && out && mean && stdv && B > 0 && C >= 1 && C <= 4 && Ho > 0 && Wo > 0, "preprocess: bad arguments");
    PreParams p;
    p.C = C; p.Ho = Ho; p.Wo = Wo;
    for (int c = 0; c < C; ++c) { p.mean[c] = mean[c]; p.stdv[c] = stdv[c]; }
    dim3 grid(cdiv(Wo, 128), Ho, B);
    preprocess_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>((const PreImage*)descs_dev, p, out);
    VD3D_CHECK_LAUNCH("preprocess");
    return VD3D_OK;
}
