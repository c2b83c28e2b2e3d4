// Stereo3D's disparity ground truth: the reference's disparity precompute (scripts/disparity_compute.py, compute_dispairity_for_split) on
// the GPU.
//   StereoBM path: cv2.StereoBM_create(192, 25).compute with cv2's defaults (XSOBEL prefilter, cap 31, texture threshold 10, uniqueness
//     15 %, no speckle filter, no left-right check, minDisparity 0) on the script's de-normalised grey frames, then the 4x4 block max of
//     the non-negative part (skimage.measure.block_reduce(.., (4, 4), np.max): far edges zero-padded).
//   LiDAR path: generate_dispariy_from_velo (R/data/kitti/utils.py:85-120): the velodyne cloud through R0_rect @ Tr_velo_to_cam and P2 in
//     float64, the last in-view point of each pixel (cloud order) giving uint16(f * baseline / depth * 16), then the same block max.
//
// Kernels:
//   bm_prefilter_kernel: the XSOBEL prefilter of both frames of a batch, from uint8 grey frames or from the float32 normalised HWC network
//     input (de-normalised and converted to grey inside the 3x3 footprint; the grey frame is written only on request).
//   stereo_bm_kernel: one CTA per (frame, strip of 64 output columns, band of 48 output rows).  The band's prefiltered rows of both frames
//     (88 left columns, 279 right columns) are staged in shared memory.  Thread i < 192 owns cost index i (disparity 191 - i) and keeps
//     the 88 vertical 25-row column sums of |P_L - P_R| in registers, sliding them one row per step; a 25-wide running sum along the strip
//     gives the row's 64 costs, stored as [i][x] in a double-buffered shared row.  Thread 192 does the same for the texture sum
//     (|P_L - 31|).  Threads 192..255 then decide one output pixel each from the 192 costs (bm_decide), while the cost threads go on
//     to the next row: one __syncthreads per row.
//   bm_border_kernel: -16 on every pixel StereoBM never computes (rows < 12 or >= H-12, columns < 203 or >= W-12).
//   disparity_block_max_kernel: the 4x4 block max of max(disp, 0) as uint16.
//   velo_scatter_kernel / velo_gather_kernel: one atomicMax of the point index per pixel (the last point in cloud order wins, as the
//     reference's sequential loop), then each pixel converts its winner's depth (or the reference's 1e9 for no point).
// The per-element routines (dg_grey, bm_prefilter_tap, bm_decide, velo_project, velo_disparity) are shared with the host entries, which
// serve as the parity checker.  Built with -fmad=false: the float64 de-normalisation and projection round every product and sum
// separately, like numpy.
#include "common.cuh"
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

namespace vd3d {

constexpr int BM_ND = 192;                      // numDisparities
constexpr int BM_HW = 12;                       // half of the 25x25 window
constexpr int BM_WIN = 2 * BM_HW + 1;
constexpr int BM_CAP = 31;                      // preFilterCap
constexpr int BM_TEXTURE = 10;                  // textureThreshold
constexpr int BM_UNIQUENESS = 15;               // uniquenessRatio (%)
constexpr int BM_FILTERED = -16;
constexpr int BM_X0 = BM_ND - 1 + BM_HW;        // 203: the first column with an output
constexpr int BM_MIN_H = 26, BM_MIN_W = 216;    // cv2 rejects H <= 25; W = 216 is the smallest width with a computed column
constexpr int BM_MAX_DIM = 1 << 14;

constexpr int BM_STRIP = 64;                    // output columns per CTA
constexpr int BM_ROWS = 48;                     // output rows per CTA
constexpr int BM_COLS = BM_STRIP + 2 * BM_HW;   // 88 column sums per cost index
constexpr int BM_RCOLS = BM_COLS + BM_ND - 1;   // 279 right-frame columns
constexpr int BM_LPITCH = BM_COLS;              // 88 (a multiple of 4: the left row is read a word at a time)
constexpr int BM_RPITCH = BM_RCOLS + 1;         // 280
constexpr int BM_IN_ROWS = BM_ROWS + 2 * BM_HW; // 72
constexpr int BM_CPITCH = BM_STRIP + 2;         // 66 halfwords per cost row: 33 words, so cost thread i's stores land on bank i + x/2
constexpr int BM_THREADS = BM_ND + BM_STRIP;    // 192 cost threads, then 64 decision threads (the first also sums the texture)
constexpr size_t BM_SMEM = (size_t)BM_IN_ROWS * (BM_LPITCH + BM_RPITCH) + 2 * BM_ND * BM_CPITCH * sizeof(uint16_t) +
                           2 * BM_STRIP * sizeof(int) + BM_COLS;

struct DenormParams { double mean[3], std[3]; };

// The script's denorm (image * rgb_std + rgb_mean in float64, clipped to [0, 1], * 255, truncated to uint8) and cv2's COLOR_BGR2GRAY on
// the result (channel 0 weighted as blue), for one pixel.
__host__ __device__ inline int dg_grey(const float* px, const DenormParams& p) {
    int c[3];
    for (int k = 0; k < 3; ++k) {
        double v = (double)px[k] * p.std[k];
        v = v + p.mean[k];
        if (v > 1) v = 1;
        if (v < 0) v = 0;
        v *= 255;
        c[k] = (int)v;
    }
    return (c[0] * 3735 + c[1] * 19235 + c[2] * 9798 + 16384) >> 15;
}

struct GreyU8 {
    const uint8_t* g; int W;
    __host__ __device__ int operator()(int x, int y) const { return g[(size_t)y * W + x]; }
    __host__ __device__ void advance(size_t pixels) { g += pixels; }
};

struct GreyF32 {
    const float* img; int W; DenormParams p;
    __host__ __device__ int operator()(int x, int y) const { return dg_grey(img + ((size_t)y * W + x) * 3, p); }
    __host__ __device__ void advance(size_t pixels) { img += pixels * 3; }
};

// cv2's XSOBEL prefilter at (x, y): clip(Sobel-x, -31, 31) + 31.  Rows reflect (row -1 reads row 1, row H reads row H-2); columns 0 and
// W-1 are 31, and so is the last row of an odd-height frame (cv2 filters rows in pairs).
template <class G>
__host__ __device__ inline uint8_t bm_prefilter_tap(const G& g, int x, int y, int H, int W) {
    if (x == 0 || x == W - 1 || ((H & 1) && y == H - 1)) return BM_CAP;
    const int yu = y > 0 ? y - 1 : 1, yd = y < H - 1 ? y + 1 : H - 2;
    int s = (g(x + 1, yu) - g(x - 1, yu)) + 2 * (g(x + 1, y) - g(x - 1, y)) + (g(x + 1, yd) - g(x - 1, yd));
    s = s < -BM_CAP ? -BM_CAP : (s > BM_CAP ? BM_CAP : s);
    return (uint8_t)(s + BM_CAP);
}

// The decision of one pixel from its 192 costs sad[i * stride] (i = 191 - d) and its texture sum: -16 for a flat window or a non-unique
// minimum, else the disparity times 16 with cv2's parabola sub-pixel step.  The first smallest cost wins (ties go to the larger disparity);
// sad[-1] reads sad[1] and sad[192] reads sad[190].
__host__ __device__ inline int16_t bm_decide(const uint16_t* sad, int stride, int texture) {
    if (texture < BM_TEXTURE) return BM_FILTERED;
    int mind = 0, minsad = sad[0];
    for (int i = 1; i < BM_ND; ++i) {
        const int v = sad[i * stride];
        if (v < minsad) { minsad = v; mind = i; }
    }
    const int thresh = minsad + minsad * BM_UNIQUENESS / 100;
    for (int j = 0; j < BM_ND; ++j)
        if ((j < mind - 1 || j > mind + 1) && sad[j * stride] <= thresh) return BM_FILTERED;
    const int p = sad[(mind < BM_ND - 1 ? mind + 1 : BM_ND - 2) * stride];
    const int n = sad[(mind > 0 ? mind - 1 : 1) * stride];
    const int den = p + n - 2 * minsad + (p > n ? p - n : n - p);
    const int d = (BM_ND - 1 - mind) * 256 + (den ? (p - n) * 256 / den : 0) + 15;
    return (int16_t)(d >> 4);
}

// generate_dispariy_from_velo's camera / image products: M = the first three rows of R0_rect @ Tr_velo_to_cam (4x4 each), P2 [3][4].
struct VeloCalib {
    double M[12], P2[12], fb;
    int H, W;
};

// One velodyne point: pts_cam = M @ [x, y, z, 1], (u, v) = (P2 @ [pts_cam, 1])[:2] / (z' + 1e-6), each sum left to right.  In view when
// 0 <= u < W-1, 0 <= v < H-1 and x > 2; then the pixel is (int(v), int(u)) and the depth pts_cam[2].
__host__ __device__ inline bool velo_project(const VeloCalib& c, const float* pt, int* px, int* py, double* depth) {
    const double x = pt[0], y = pt[1], z = pt[2];
    double cam[3], pix[3];
    for (int r = 0; r < 3; ++r) cam[r] = c.M[r * 4] * x + c.M[r * 4 + 1] * y + c.M[r * 4 + 2] * z + c.M[r * 4 + 3];
    for (int r = 0; r < 3; ++r) pix[r] = c.P2[r * 4] * cam[0] + c.P2[r * 4 + 1] * cam[1] + c.P2[r * 4 + 2] * cam[2] + c.P2[r * 4 + 3];
    const double u = pix[0] / (pix[2] + 1e-6), v = pix[1] / (pix[2] + 1e-6);
    if (!(u < c.W - 1 && u >= 0 && v < c.H - 1 && v >= 0 && x > 2)) return false;
    *px = (int)u;
    *py = (int)v;
    *depth = cam[2];
    return true;
}

// (P2[0, 0] * baseline) / depth * 16 as uint16 (truncated); an empty pixel has the reference's depth 1e9.  Values outside the int32 range
// give 0; within it the low 16 bits, as the reference's cast does on x86.
__host__ __device__ inline uint16_t velo_disparity(double fb, double depth) {
    const double d = fb / depth * 16;
    if (!(d > -2147483648.0 && d < 2147483648.0)) return 0;
    return (uint16_t)(int)d;
}

// ---- kernels ------------------------------------------------------------------------------------------------------------------------

template <class G>
__global__ void bm_prefilter_kernel(G gl, G gr, int B, int H, int W, uint8_t* planes, uint8_t* grey) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    const int f = blockIdx.z;                                   // frame: left images 0..B-1, then right images
    if (x >= W) return;
    G g = f < B ? gl : gr;
    const size_t off = (size_t)(f < B ? f : f - B) * H * W;
    g.advance(off);
    const size_t o = (size_t)f * H * W + (size_t)y * W + x;
    planes[o] = bm_prefilter_tap(g, x, y, H, W);
    if (grey) grey[o] = (uint8_t)g(x, y);
}

__global__ void bm_border_kernel(int B, int H, int W, int16_t* disp) {
    const long long n = (long long)B * H * W;
    for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(k % W), y = (int)(k / W % H);
        if (y < BM_HW || y >= H - BM_HW || x < BM_X0 || x >= W - BM_HW) disp[k] = BM_FILTERED;
    }
}

__global__ void __launch_bounds__(BM_THREADS, 2) stereo_bm_kernel(const uint8_t* planes, int B, int H, int W, int16_t* disp) {
    extern __shared__ __align__(16) uint8_t sm[];
    uint8_t* sl = sm;                                               // [BM_IN_ROWS][BM_LPITCH]
    uint8_t* sr = sl + BM_IN_ROWS * BM_LPITCH;                      // [BM_IN_ROWS][BM_RPITCH]
    uint16_t* scost = (uint16_t*)(sr + BM_IN_ROWS * BM_RPITCH);     // [2][BM_ND][BM_CPITCH]
    int* stex = (int*)(scost + 2 * BM_ND * BM_CPITCH);              // [2][BM_STRIP]
    uint8_t* s31 = (uint8_t*)(stex + 2 * BM_STRIP);                 // [BM_COLS] of 31: the texture thread's "right frame"

    const int t = threadIdx.x, b = blockIdx.z;
    const int x0 = BM_X0 + blockIdx.x * BM_STRIP, y0 = BM_HW + blockIdx.y * BM_ROWS;
    const int nx = min(BM_STRIP, W - BM_HW - x0), ny = min(BM_ROWS, H - BM_HW - y0);
    const int lc0 = x0 - BM_HW, rc0 = lc0 - (BM_ND - 1), r0 = y0 - BM_HW, nr = ny + 2 * BM_HW;
    const uint8_t* L = planes + (size_t)b * H * W;
    const uint8_t* R = planes + ((size_t)B + b) * H * W;
    for (int k = t; k < nr * BM_LPITCH; k += BM_THREADS) {
        const int r = k / BM_LPITCH, x = lc0 + k % BM_LPITCH;
        sl[k] = x < W ? L[(size_t)(r0 + r) * W + x] : 0;         // columns past W-1 feed only outputs past W-13, which are not written
    }
    for (int k = t; k < nr * BM_RPITCH; k += BM_THREADS) {
        const int r = k / BM_RPITCH, c = k % BM_RPITCH, x = rc0 + c;
        sr[k] = c < BM_RCOLS && x < W ? R[(size_t)(r0 + r) * W + x] : 0;
    }
    for (int k = t; k < BM_COLS; k += BM_THREADS) s31[k] = BM_CAP;
    __syncthreads();

    const bool summer = t <= BM_ND;                                 // cost threads and the texture thread
    const int i = t < BM_ND ? t : 0;
    const int rpitch = t < BM_ND ? BM_RPITCH : 0;
    const uint8_t* rbase = t < BM_ND ? sr + i : s31;
    int V[BM_COLS];
    auto slide = [&](int r, bool add) {
        const uint8_t* lrow = sl + r * BM_LPITCH;
        const uint8_t* rrow = rbase + r * rpitch;
#pragma unroll
        for (int c = 0; c < BM_COLS; c += 4) {
            const uint32_t lw = *(const uint32_t*)(lrow + c);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const unsigned a = (lw >> (8 * j)) & 255u, s = __usad(a, rrow[c + j], 0u);
                V[c + j] = add ? V[c + j] + (int)s : V[c + j] - (int)s;
            }
        }
    };
    if (summer) {
#pragma unroll
        for (int c = 0; c < BM_COLS; ++c) V[c] = 0;
        for (int r = 0; r < 2 * BM_HW; ++r) slide(r, true);
    }
    for (int yy = 0; yy < ny; ++yy) {
        uint16_t* cb = scost + (yy & 1) * BM_ND * BM_CPITCH;
        int* tb = stex + (yy & 1) * BM_STRIP;
        if (summer) {
            slide(yy + 2 * BM_HW, true);                            // the window now holds rows y-12 .. y+12
            int s = 0;
#pragma unroll
            for (int c = 0; c < BM_WIN; ++c) s += V[c];
#pragma unroll
            for (int x = 0; x < BM_STRIP; ++x) {
                if (t < BM_ND) cb[i * BM_CPITCH + x] = (uint16_t)s;
                else tb[x] = s;
                if (x + 1 < BM_STRIP) s += V[x + BM_WIN] - V[x];
            }
            slide(yy, false);                                       // drop row y-12
        }
        __syncthreads();
        const int x = t - BM_ND;
        if (x >= 0 && x < nx)
            disp[((size_t)b * H + y0 + yy) * W + x0 + x] = bm_decide(cb + x, BM_CPITCH, tb[x]);
    }
}

template <class T>
__global__ void disparity_block_max_kernel(const T* in, int B, int H, int W, uint16_t* out) {
    const int Ho = (H + 3) / 4, Wo = (W + 3) / 4;
    const long long n = (long long)B * Ho * Wo;
    for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
        const int ox = (int)(k % Wo), oy = (int)(k / Wo % Ho), b = (int)(k / ((long long)Wo * Ho));
        int m = 0;
        for (int y = oy * 4; y < min(oy * 4 + 4, H); ++y)
            for (int x = ox * 4; x < min(ox * 4 + 4, W); ++x) m = max(m, (int)in[((size_t)b * H + y) * W + x]);
        out[k] = (uint16_t)m;
    }
}

__global__ void velo_scatter_kernel(const float* pts, int N, int stride, VeloCalib c, int* winner) {
    for (int n = blockIdx.x * blockDim.x + threadIdx.x; n < N; n += gridDim.x * blockDim.x) {
        int px, py;
        double depth;
        if (velo_project(c, pts + (size_t)n * stride, &px, &py, &depth)) atomicMax(winner + (size_t)py * c.W + px, n);
    }
}

__global__ void velo_gather_kernel(const float* pts, int stride, VeloCalib c, const int* winner, uint16_t* full) {
    const int n = c.H * c.W;
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
        const int w = winner[k];
        double depth = 1e9;
        int px, py;
        if (w >= 0) velo_project(c, pts + (size_t)w * stride, &px, &py, &depth);
        full[k] = velo_disparity(c.fb, depth);
    }
}

// ---- host side ----------------------------------------------------------------------------------------------------------------------

static int check_bm_shape(int B, int H, int W, const char* who) {
    VD3D_REQUIRE(B > 0 && B <= 65535, "%s: batch %d outside [1, 65535]", who, B);
    VD3D_REQUIRE(H >= BM_MIN_H && W >= BM_MIN_W && H <= BM_MAX_DIM && W <= BM_MAX_DIM,
                 "%s: %dx%d frame outside [%d, %d] x [%d, %d] (StereoBM(192, 25) has no defined output below %dx%d)", who, H, W, BM_MIN_H,
                 BM_MAX_DIM, BM_MIN_W, BM_MAX_DIM, BM_MIN_H, BM_MIN_W);
    return VD3D_OK;
}

static int check_dims(int B, int H, int W, const char* who) {
    VD3D_REQUIRE(B > 0 && B <= 65535 && H > 0 && W > 0 && H <= BM_MAX_DIM && W <= BM_MAX_DIM, "%s: bad shape %dx%dx%d", who, B, H, W);
    return VD3D_OK;
}

static DenormParams denorm_params(const double* mean, const double* std) {
    DenormParams p;
    for (int k = 0; k < 3; ++k) { p.mean[k] = mean[k]; p.std[k] = std[k]; }
    return p;
}

static int velo_calib(const double* R0, const double* Tr, const double* P2, double baseline, int H, int W, VeloCalib* c) {
    for (int k = 0; k < 16; ++k) VD3D_REQUIRE(isfinite(R0[k]) && isfinite(Tr[k]), "velo_disparity: R0_rect / Tr_velo_to_cam not finite");
    for (int k = 0; k < 12; ++k) VD3D_REQUIRE(isfinite(P2[k]), "velo_disparity: P2 not finite");
    VD3D_REQUIRE(isfinite(baseline), "velo_disparity: baseline not finite");
    for (int r = 0; r < 3; ++r)
        for (int k = 0; k < 4; ++k)
            c->M[r * 4 + k] = R0[r * 4] * Tr[k] + R0[r * 4 + 1] * Tr[4 + k] + R0[r * 4 + 2] * Tr[8 + k] + R0[r * 4 + 3] * Tr[12 + k];
    for (int k = 0; k < 12; ++k) c->P2[k] = P2[k];
    c->fb = P2[0] * baseline;
    c->H = H;
    c->W = W;
    return VD3D_OK;
}

// The prefilter, border and block-matching launches over planes [2][B][H][W] already holding (or about to hold, in stream order) the
// prefiltered frames.
static int bm_launch(const uint8_t* planes, int B, int H, int W, int16_t* disp, cudaStream_t st) {
    static bool attr = false;
    if (!attr) {
        VD3D_CUDA(cudaFuncSetAttribute(stereo_bm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BM_SMEM));
        attr = true;
    }
    const long long n = (long long)B * H * W;
    bm_border_kernel<<<(int)std::min<long long>(cdiv(n, 256), 4 * kNumSMs * 8), 256, 0, st>>>(B, H, W, disp);
    VD3D_CHECK_LAUNCH("bm_border");
    dim3 grid(cdiv(W - BM_HW - BM_X0, BM_STRIP), cdiv(H - 2 * BM_HW, BM_ROWS), B);
    stereo_bm_kernel<<<grid, BM_THREADS, BM_SMEM, st>>>(planes, B, H, W, disp);
    VD3D_CHECK_LAUNCH("stereo_bm");
    return VD3D_OK;
}

}  // namespace vd3d

using namespace vd3d;

// ---- device entries -----------------------------------------------------------------------------------------------------------------

extern "C" long long vd3d_stereo_bm_workspace_bytes(int B, int H, int W) {
    if (check_bm_shape(B, H, W, "stereo_bm_workspace_bytes")) return VD3D_EINVAL;
    return 2LL * B * H * W;
}

extern "C" int vd3d_stereo_bm(const uint8_t* left, const uint8_t* right, int B, int H, int W, uint8_t* workspace, int16_t* disp,
                              void* stream) {
    VD3D_REQUIRE(left && right && workspace && disp, "stereo_bm: null argument");
    int rc = check_bm_shape(B, H, W, "stereo_bm");
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    bm_prefilter_kernel<GreyU8><<<dim3(cdiv(W, 128), H, 2 * B), 128, 0, st>>>(GreyU8{left, W}, GreyU8{right, W}, B, H, W, workspace, nullptr);
    VD3D_CHECK_LAUNCH("bm_prefilter_u8");
    return bm_launch(workspace, B, H, W, disp, st);
}

extern "C" int vd3d_stereo_bm_f32(const float* left, const float* right, int B, int H, int W, const double* mean_host,
                                  const double* std_host, uint8_t* workspace, uint8_t* grey, int16_t* disp, void* stream) {
    VD3D_REQUIRE(left && right && mean_host && std_host && workspace && disp, "stereo_bm_f32: null argument");
    int rc = check_bm_shape(B, H, W, "stereo_bm_f32");
    if (rc) return rc;
    const DenormParams p = denorm_params(mean_host, std_host);
    cudaStream_t st = (cudaStream_t)stream;
    bm_prefilter_kernel<GreyF32><<<dim3(cdiv(W, 128), H, 2 * B), 128, 0, st>>>(GreyF32{left, W, p}, GreyF32{right, W, p}, B, H, W, workspace,
                                                                                grey);
    VD3D_CHECK_LAUNCH("bm_prefilter_f32");
    return bm_launch(workspace, B, H, W, disp, st);
}

extern "C" int vd3d_disparity_block_max(const void* in, int is_signed, int B, int H, int W, uint16_t* out, void* stream) {
    VD3D_REQUIRE(in && out, "disparity_block_max: null argument");
    int rc = check_dims(B, H, W, "disparity_block_max");
    if (rc) return rc;
    const long long n = (long long)B * ((H + 3) / 4) * ((W + 3) / 4);
    const int grid = (int)std::min<long long>(cdiv(n, 256), 4 * kNumSMs * 8);
    if (is_signed) disparity_block_max_kernel<int16_t><<<grid, 256, 0, (cudaStream_t)stream>>>((const int16_t*)in, B, H, W, out);
    else disparity_block_max_kernel<uint16_t><<<grid, 256, 0, (cudaStream_t)stream>>>((const uint16_t*)in, B, H, W, out);
    VD3D_CHECK_LAUNCH("disparity_block_max");
    return VD3D_OK;
}

extern "C" int vd3d_velo_disparity(const float* points, int N, int stride, const double* R0_host, const double* Tr_host,
                                   const double* P2_host, double baseline, int H, int W, int* winner, uint16_t* full, void* stream) {
    VD3D_REQUIRE(points && R0_host && Tr_host && P2_host && winner && full, "velo_disparity: null argument");
    VD3D_REQUIRE(N >= 0 && stride >= 3, "velo_disparity: %d points of stride %d", N, stride);
    int rc = check_dims(1, H, W, "velo_disparity");
    if (rc) return rc;
    VeloCalib c;
    rc = velo_calib(R0_host, Tr_host, P2_host, baseline, H, W, &c);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    VD3D_CUDA(cudaMemsetAsync(winner, 0xff, (size_t)H * W * sizeof(int), st));
    if (N > 0) {
        velo_scatter_kernel<<<std::min(cdiv(N, 256), 8 * kNumSMs), 256, 0, st>>>(points, N, stride, c, winner);
        VD3D_CHECK_LAUNCH("velo_scatter");
    }
    velo_gather_kernel<<<std::min(cdiv((long long)H * W, 256), 8 * kNumSMs), 256, 0, st>>>(points, stride, c, winner, full);
    VD3D_CHECK_LAUNCH("velo_gather");
    return VD3D_OK;
}

// ---- host entries (the parity checker; same routines, one frame) --------------------------------------------------------------------

extern "C" int vd3d_disparity_grey_host(const float* img, int H, int W, const double* mean, const double* std, uint8_t* grey) {
    VD3D_REQUIRE(img && mean && std && grey, "disparity_grey_host: null argument");
    int rc = check_dims(1, H, W, "disparity_grey_host");
    if (rc) return rc;
    const DenormParams p = denorm_params(mean, std);
    for (size_t k = 0; k < (size_t)H * W; ++k) grey[k] = (uint8_t)dg_grey(img + 3 * k, p);
    return VD3D_OK;
}

extern "C" int vd3d_stereo_bm_host(const uint8_t* left, const uint8_t* right, int H, int W, int16_t* disp) {
    VD3D_REQUIRE(left && right && disp, "stereo_bm_host: null argument");
    int rc = check_bm_shape(1, H, W, "stereo_bm_host");
    if (rc) return rc;
    std::vector<uint8_t> pl((size_t)H * W), pr((size_t)H * W);
    for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x) {
            pl[(size_t)y * W + x] = bm_prefilter_tap(GreyU8{left, W}, x, y, H, W);
            pr[(size_t)y * W + x] = bm_prefilter_tap(GreyU8{right, W}, x, y, H, W);
        }
    for (size_t k = 0; k < (size_t)H * W; ++k) disp[k] = BM_FILTERED;
    // col[i][x]: the 25-row sum of |P_L(x) - P_R(x - d)| (i = ND-1-d; i = ND: |P_L - 31|, the texture) for the current output row
    std::vector<int> col((size_t)(BM_ND + 1) * W, 0);
    std::vector<uint16_t> sad((size_t)W * BM_ND);
    std::vector<int> tex(W);
    auto add_row = [&](int y, int sign) {
        const uint8_t* a = &pl[(size_t)y * W];
        const uint8_t* b = &pr[(size_t)y * W];
        for (int i = 0; i <= BM_ND; ++i) {
            const int d = BM_ND - 1 - i;
            int* c = &col[(size_t)i * W];
            for (int x = BM_X0 - BM_HW; x < W; ++x) c[x] += sign * abs((int)a[x] - (i < BM_ND ? (int)b[x - d] : BM_CAP));
        }
    };
    for (int y = 0; y < 2 * BM_HW; ++y) add_row(y, 1);
    for (int y = BM_HW; y < H - BM_HW; ++y) {
        add_row(y + BM_HW, 1);
        for (int i = 0; i <= BM_ND; ++i) {
            const int* c = &col[(size_t)i * W];
            int s = 0;
            for (int x = BM_X0 - BM_HW; x < BM_X0 + BM_HW + 1; ++x) s += c[x];
            for (int x = BM_X0; x < W - BM_HW; ++x) {
                if (i < BM_ND) sad[(size_t)x * BM_ND + i] = (uint16_t)s;
                else tex[x] = s;
                if (x + BM_HW + 1 < W) s += c[x + BM_HW + 1] - c[x - BM_HW];
            }
        }
        for (int x = BM_X0; x < W - BM_HW; ++x) disp[(size_t)y * W + x] = bm_decide(&sad[(size_t)x * BM_ND], 1, tex[x]);
        add_row(y - BM_HW, -1);
    }
    return VD3D_OK;
}

extern "C" int vd3d_disparity_block_max_host(const void* in, int is_signed, int H, int W, uint16_t* out) {
    VD3D_REQUIRE(in && out, "disparity_block_max_host: null argument");
    int rc = check_dims(1, H, W, "disparity_block_max_host");
    if (rc) return rc;
    const int Ho = (H + 3) / 4, Wo = (W + 3) / 4;
    for (int oy = 0; oy < Ho; ++oy)
        for (int ox = 0; ox < Wo; ++ox) {
            int m = 0;
            for (int y = oy * 4; y < std::min(oy * 4 + 4, H); ++y)
                for (int x = ox * 4; x < std::min(ox * 4 + 4, W); ++x) {
                    const size_t k = (size_t)y * W + x;
                    m = std::max(m, is_signed ? (int)((const int16_t*)in)[k] : (int)((const uint16_t*)in)[k]);
                }
            out[(size_t)oy * Wo + ox] = (uint16_t)m;
        }
    return VD3D_OK;
}

extern "C" int vd3d_velo_disparity_host(const float* points, int N, int stride, const double* R0, const double* Tr, const double* P2,
                                        double baseline, int H, int W, uint16_t* full) {
    VD3D_REQUIRE(points && R0 && Tr && P2 && full, "velo_disparity_host: null argument");
    VD3D_REQUIRE(N >= 0 && stride >= 3, "velo_disparity_host: %d points of stride %d", N, stride);
    int rc = check_dims(1, H, W, "velo_disparity_host");
    if (rc) return rc;
    VeloCalib c;
    rc = velo_calib(R0, Tr, P2, baseline, H, W, &c);
    if (rc) return rc;
    std::vector<double> depth((size_t)H * W, 1e9);
    for (int n = 0; n < N; ++n) {
        int px, py;
        double z;
        if (velo_project(c, points + (size_t)n * stride, &px, &py, &z)) depth[(size_t)py * W + px] = z;
    }
    for (size_t k = 0; k < (size_t)H * W; ++k) full[k] = velo_disparity(c.fb, depth[k]);
    return VD3D_OK;
}
