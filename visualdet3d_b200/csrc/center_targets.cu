// CenterNet-style training targets of KM3D and MonoFlex: the reference's KittiRTM3DDataset._build_target and
// KittiMonoFlexDataset._build_target (R/data/kitti/dataset/KM3D_dataset.py:57-221, 346-527) with BBox3dProjector
// (R/networks/utils/utils.py:222-253), theta2alpha_3d / alpha2theta_3d (R/utils/utils.py:47-79) and gaussian_radius / gaussian2D /
// gen_hm_radius (R/networks/utils/rtm3d_utils.py:52-109).
//
// Two launches per batch, no host synchronisation:
//   per-object pass: one warp per image, one lane per object slot (max_objects = 32).  Each lane writes every sparse target of its slot
//     (zeros included) and its splats (channel, integer centre, radius) into the image's fixed splat slots;
//   heatmap render: a gather-max over the image's splats.  Every heatmap element is written once, zeros included: no memset, no atomic,
//     the same bits on every run.
// The per-object routine (ct_object) and the per-pixel routine (ct_pixel) are shared with the host entry (vd3d_center_targets_host: the
// parity checker).  Arithmetic follows the reference's types: float64 where it uses numpy float64 (theta2alpha_3d, the bbox clip,
// gaussian_radius, rotbin / rotres, rots, the Gaussian), float32 where it uses torch float32 (the projector), in the reference's order of
// operations.  atan2 / sin / cos of the float32 projector are evaluated in float64 and rounded, so the host and the device agree bit for
// bit; torch's CPU float32 kernels may differ from that by an ulp.  Built with -fmad=false: every product and sum rounds separately.
#include "common.cuh"
#include <float.h>
#include <limits.h>
#include <string.h>
#include <math.h>

namespace vd3d {

constexpr int CT_MAX_OBJ = 32;
constexpr int CT_MAX_VERT = 10;
constexpr int CT_MAX_CLASSES = 64;
constexpr int CT_SCALE = 4;
constexpr int CT_SPLATS = CT_MAX_OBJ * (1 + CT_MAX_VERT);
constexpr int CT_FIELDS = 11;                           // x, y, z, w, h, l, ry, bbox_l, bbox_t, bbox_r, bbox_b
enum { CT_KM3D = 0, CT_MONOFLEX = 1 };

// Output slots (vd3d_center_targets / _host `outs`): the reference's targets, plus the splat list of the device form.
enum {
    O_HM, O_HM_HP, O_HPS, O_REG, O_HP_OFFSET, O_DIM, O_ROTS, O_ROTBIN, O_ROTRES, O_DEP, O_IND, O_HP_IND, O_REG_MASK, O_HPS_MASK,
    O_HP_MASK, O_WH, O_LOCATION, O_ORI, O_KP_DEPTH_MASK, O_BBOXES2D, O_BBOXES2D_TARGET, CT_NOUT
};

struct CtRecord {
    double P2[12];
    double obj[CT_MAX_OBJ][CT_FIELDS];
    int cls[CT_MAX_OBJ];
    int n, mode, img_h, img_w, num_classes, pad;
};

struct CtOut { void* p[CT_NOUT]; };

struct CtShape {
    int mode, K, C, hm_h, hm_w;
};

__host__ __device__ inline CtShape ct_shape(int mode, int img_h, int img_w, int num_classes) {
    CtShape s;
    s.mode = mode; s.K = mode == CT_MONOFLEX ? 10 : 9; s.C = num_classes;
    s.hm_h = img_h / CT_SCALE; s.hm_w = img_w / CT_SCALE;
    return s;
}

// One splat of gen_hm_radius: channel (class, or num_classes + vertex), integer centre, radius; r < 0: none.
struct CtSplat { int c, x, y, r; };

// gaussian_radius((ceil(bbox_h), ceil(bbox_w)), 0.7) in float64, the reference's expressions in its order
__host__ __device__ inline double ct_gaussian_radius(double height, double width) {
    const double mo = 0.7;
    const double b1 = height + width;
    const double c1 = width * height * (1 - mo) / (1 + mo);
    const double sq1 = sqrt(b1 * b1 - 4 * c1);
    const double r1 = (b1 + sq1) / 2;
    const double b2 = 2 * (height + width);
    const double c2 = (1 - mo) * width * height;
    const double sq2 = sqrt(b2 * b2 - 16 * c2);
    const double r2 = (b2 + sq2) / 2;
    const double a3 = 4 * mo;
    const double b3 = -2 * mo * (height + width);
    const double c3 = (mo - 1) * width * height;
    const double sq3 = sqrt(b3 * b3 - 4 * a3 * c3);
    const double r3 = (b3 + sq3) / 2;
    return fmin(r1, fmin(r2, r3));
}

// `float.astype(np.int32)`: truncation toward zero; NaN and values outside int32 give INT_MIN, as x86's cvttss2si does
__host__ __device__ inline int ct_trunc(float v) { return (v > -2147483648.f && v < 2147483648.f) ? (int)v : INT_MIN; }

template <typename T>
__host__ __device__ inline T* ct_at(const CtOut& o, int slot, size_t off) { return (T*)o.p[slot] + off; }

// Every sparse target of object slot k of image b, and its splats.  `o` holds the batch's arrays ([B, ...]); the host form passes b == 0.
// The slot is zero-filled first, then the reference's assignments are replayed in its order.
__host__ __device__ inline void ct_object(const CtRecord& rec, const CtShape& s, int b, int k, const CtOut& o, CtSplat* splats) {
    const int K = s.K;
    const size_t kb = (size_t)b * CT_MAX_OBJ + k;
    float* hps = ct_at<float>(o, O_HPS, kb * 2 * K);
    float* hp_off = ct_at<float>(o, O_HP_OFFSET, kb * 2 * K);
    unsigned char* hps_mask = ct_at<unsigned char>(o, O_HPS_MASK, kb * 2 * K);
    long long* hp_ind = ct_at<long long>(o, O_HP_IND, kb * K);
    unsigned char* hp_mask = ct_at<unsigned char>(o, O_HP_MASK, kb * K);
    float* reg = ct_at<float>(o, O_REG, kb * 2);
    float* rots = ct_at<float>(o, O_ROTS, kb * 2);
    long long* rotbin = ct_at<long long>(o, O_ROTBIN, kb * 2);
    float* rotres = ct_at<float>(o, O_ROTRES, kb * 2);
    float* wh = ct_at<float>(o, O_WH, kb * 2);
    float* dim = ct_at<float>(o, O_DIM, kb * 3);
    float* loc = ct_at<float>(o, O_LOCATION, kb * 3);
    float* dep = ct_at<float>(o, O_DEP, kb);
    float* ori = ct_at<float>(o, O_ORI, kb);
    long long* ind = ct_at<long long>(o, O_IND, kb);
    unsigned char* reg_mask = ct_at<unsigned char>(o, O_REG_MASK, kb);
    const bool mf = s.mode == CT_MONOFLEX;
    float* kpd = mf ? ct_at<float>(o, O_KP_DEPTH_MASK, kb * 3) : nullptr;
    float* bb2d = mf ? ct_at<float>(o, O_BBOXES2D, kb * 4) : nullptr;
    float* bbt = mf ? ct_at<float>(o, O_BBOXES2D_TARGET, kb * 4) : nullptr;
    for (int j = 0; j < 2 * K; ++j) { hps[j] = 0.f; hp_off[j] = 0.f; hps_mask[j] = 0; }
    for (int j = 0; j < K; ++j) { hp_ind[j] = 0; hp_mask[j] = 0; }
    for (int i = 0; i < 2; ++i) { reg[i] = 0.f; rots[i] = 0.f; rotbin[i] = 0; rotres[i] = 0.f; wh[i] = 0.f; }
    for (int i = 0; i < 3; ++i) { dim[i] = 0.f; loc[i] = 0.f; }
    *dep = 0.f; *ori = 0.f; *ind = 0; *reg_mask = 0;
    if (mf) {
        for (int i = 0; i < 3; ++i) kpd[i] = 0.f;
        for (int i = 0; i < 4; ++i) { bb2d[i] = 0.f; bbt[i] = 0.f; }
    }
    CtSplat* sp = splats + k * (1 + K);
    for (int j = 0; j <= K; ++j) sp[j].r = -1;
    if (k >= rec.n) return;

    const double* ob = rec.obj[k];
    const double x = ob[0], y = ob[1], z = ob[2], w = ob[3], h = ob[4], l = ob[5], ry = ob[6];
    const double* P = rec.P2;
    const double alpha = ry - atan2(x + P[3] / P[0], z);          // theta2alpha_3d on the float64 P2
    *ori = (float)ry;
    const double sa = sin(alpha);
    if (sa < 0.5) { rotbin[0] = 1; rotres[0] = (float)(alpha - (-0.5 * M_PI)); }
    if (sa > -0.5) { rotbin[1] = 1; rotres[1] = (float)(alpha - (0.5 * M_PI)); }
    double bb[4] = {ob[7] / CT_SCALE, ob[8] / CT_SCALE, ob[9] / CT_SCALE, ob[10] / CT_SCALE};
    if (mf)
        for (int i = 0; i < 4; ++i) bb2d[i] = (float)bb[i];      // unclipped, for every object
    const double xmax = (double)(rec.img_w / CT_SCALE), ymax = (double)(rec.img_h / CT_SCALE);
    bb[0] = fmin(fmax(bb[0], 0.0), xmax); bb[2] = fmin(fmax(bb[2], 0.0), xmax);
    bb[1] = fmin(fmax(bb[1], 0.0), ymax); bb[3] = fmin(fmax(bb[3], 0.0), ymax);
    const double bbox_h = bb[3] - bb[1], bbox_w = bb[2] - bb[0];
    if (!(bbox_h > 0 && bbox_w > 0)) return;

    // bbox3d_origin's row (torch float32) and BBox3dProjector.forward
    const float xf = (float)x, yf = (float)(y - 0.5 * h), zf = (float)z;
    const float dims[3] = {(float)w, (float)h, (float)l};
    loc[0] = xf; loc[1] = yf; loc[2] = zf;                      // written before the centre's range check
    float Pf[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) Pf[i] = (float)P[i];
    const float theta = (float)alpha + (float)atan2((double)(xf + Pf[3] / Pf[0]), (double)zf);
    const float c = (float)cos((double)theta), sn = (float)sin((double)theta);
    float vx[11], vy[11], vz[11];
#pragma unroll
    for (int j = 0; j < 11; ++j) {
        // corner_matrix rows 0..7: x -1 1 1 1 1 -1 -1 -1, y -1 -1 1 1 -1 -1 1 1, z -1 -1 -1 1 1 1 1 -1; then KM3D's row 8 = the centre,
        // MonoFlex's rows 8, 9, 10 = (0, 1, 0), (0, -1, 0), the centre
        const float cm0 = (j >= 1 && j <= 4) ? 1.f : j < 8 ? -1.f : 0.f;
        const float cm1 = (j == 2 || j == 3 || j == 6 || j == 7) ? 1.f : j < 8 ? -1.f : (mf && j == 8) ? 1.f : (mf && j == 9) ? -1.f : 0.f;
        const float cm2 = (j >= 3 && j <= 6) ? 1.f : j < 8 ? -1.f : 0.f;
        const float r0 = (0.5f * cm0) * dims[0], r1 = (0.5f * cm1) * dims[1], r2 = (0.5f * cm2) * dims[2];
        const float ax = (r2 * c + r0 * sn) + xf, ay = r1 + yf, az = (-r2 * sn + r0 * c) + zf;
        const float c0 = ((Pf[0] * ax + Pf[1] * ay) + Pf[2] * az) + Pf[3];
        const float c1 = ((Pf[4] * ax + Pf[5] * ay) + Pf[6] * az) + Pf[7];
        const float c2 = ((Pf[8] * ax + Pf[9] * ay) + Pf[10] * az) + Pf[11];
        const float den = c2 + 1e-6f;
        vx[j] = c0 / den / (float)CT_SCALE;
        vy[j] = c1 / den / (float)CT_SCALE;
        vz[j] = az;
    }
    const int rg = (int)ct_gaussian_radius(ceil(bbox_h), ceil(bbox_w));
    const int radius = rg > 0 ? rg : 0;
    float cx, cy;
    bool kv[3] = {false, false, false};
    if (mf) {
        // keypoint visibility: inside [0, hm_w] x [0, hm_h] (inclusive) and in front of the camera; only kp_detph_mask reads it
        bool vis[10];
#pragma unroll
        for (int j = 0; j < 10; ++j) vis[j] = vx[j] >= 0 && vx[j] <= (float)s.hm_w && vy[j] >= 0 && vy[j] <= (float)s.hm_h && vz[j] > 0;
        bool v2[10];
#pragma unroll
        for (int j = 0; j < 8; ++j) v2[j] = vis[j & 3] || vis[(j & 3) + 4];
        v2[8] = v2[9] = vis[8] || vis[9];
        kv[0] = v2[8] && v2[9];
        kv[1] = v2[0] && v2[2] && v2[4] && v2[6];
        kv[2] = v2[1] && v2[3] && v2[5] && v2[7];
        cx = vx[10]; cy = vy[10];                                 // the projected box centre
    } else {
        cx = (float)((bb[0] + bb[2]) / 2); cy = (float)((bb[1] + bb[3]) / 2);
    }
    const int cix = ct_trunc(cx), ciy = ct_trunc(cy);
    if (!(0 <= cix && cix < s.hm_w && 0 <= ciy && ciy < s.hm_h)) return;

    sp[0] = CtSplat{rec.cls[k], cix, ciy, radius};
    *ind = (long long)ciy * s.hm_w + cix;
#pragma unroll
    for (int j = 0; j < CT_MAX_VERT; ++j) {
        if (j >= K) break;
        const int vix = ct_trunc(vx[j]), viy = ct_trunc(vy[j]);
        hps[2 * j] = vx[j] - (float)cix;
        hps[2 * j + 1] = vy[j] - (float)ciy;
        hps_mask[2 * j] = hps_mask[2 * j + 1] = 1;
        if (0 <= vix && vix < s.hm_w && 0 <= viy && viy < s.hm_h) {
            sp[1 + j] = CtSplat{s.C + j, vix, viy, radius};
            hp_off[2 * j] = vx[j] - (float)vix;
            hp_off[2 * j + 1] = vy[j] - (float)viy;
            hp_mask[j] = 1;
            hp_ind[j] = (long long)viy * s.hm_w + vix;
        }
    }
    reg[0] = cx - (float)cix; reg[1] = cy - (float)ciy;
    if (mf) {
        bbt[0] = (float)(cix - bb[0]); bbt[1] = (float)(ciy - bb[1]);
        bbt[2] = (float)(bb[2] - cix); bbt[3] = (float)(bb[3] - ciy);
    }
    dim[0] = (float)w; dim[1] = (float)h; dim[2] = (float)l;
    rots[0] = (float)sin(alpha); rots[1] = (float)cos(alpha);
    *dep = (float)z;
    wh[0] = (float)bbox_w; wh[1] = (float)bbox_h;
    *reg_mask = 1;
    if (mf)
        for (int i = 0; i < 3; ++i) kpd[i] = kv[i] ? 1.f : 0.f;
}

// gaussian2D((2r+1, 2r+1), sigma=(2r+1)/6) at offset (dx, dy), float64, zeroed below eps * max (max == exp(0) == 1)
__host__ __device__ inline double ct_gauss(int dx, int dy, int r) {
    const double sigma = (double)(2 * r + 1) / 6;
    const double xx = (double)dx, yy = (double)dy;
    const double g = exp(-(xx * xx + yy * yy) / (2 * sigma * sigma));
    return g < DBL_EPSILON ? 0.0 : g;
}

// One heatmap element: the max over the splats of its channel (np.maximum into a zero float32 map: the float64 value rounded on store)
__host__ __device__ inline float ct_pixel(const CtSplat* sp, int n, int x, int y) {
    float v = 0.f;
    for (int i = 0; i < n; ++i) {
        const int dx = x - sp[i].x, dy = y - sp[i].y, r = sp[i].r;
        if (dx >= -r && dx <= r && dy >= -r && dy <= r) v = fmaxf(v, (float)ct_gauss(dx, dy, r));
    }
    return v;
}

constexpr int CT_OBJ_WARPS = 4;

__global__ void __launch_bounds__(CT_OBJ_WARPS * 32) center_targets_object_kernel(const CtRecord* __restrict__ recs, int B, CtShape s,
                                                                                   CtOut o, CtSplat* __restrict__ splats) {
    const int b = blockIdx.x * CT_OBJ_WARPS + threadIdx.x / 32;
    if (b >= B) return;
    ct_object(recs[b], s, b, threadIdx.x & 31, o, splats + (size_t)b * CT_SPLATS);
}

constexpr int CT_RENDER_THREADS = 128;
constexpr int CT_RENDER_ROWS = 8;

// grid (row bands, channels, images).  The block first gathers the splats of its channel that reach its rows (at most 32 per channel:
// one per object), then writes every element of its rows, four columns per thread (a 16-byte store when rows are 16-byte aligned).
__global__ void __launch_bounds__(CT_RENDER_THREADS) center_targets_render_kernel(const CtSplat* __restrict__ splats, CtShape s,
                                                                                  float* __restrict__ hm, float* __restrict__ hm_hp) {
    __shared__ CtSplat sh[CT_MAX_OBJ];
    __shared__ int cnt;
    const int b = blockIdx.z, ch = blockIdx.y, y0 = blockIdx.x * CT_RENDER_ROWS;
    const int y1 = min(y0 + CT_RENDER_ROWS, s.hm_h) - 1;
    const int nslot = CT_MAX_OBJ * (1 + s.K);
    if (threadIdx.x == 0) cnt = 0;
    __syncthreads();
    const CtSplat* src = splats + (size_t)b * CT_SPLATS;
    for (int i = threadIdx.x; i < nslot; i += CT_RENDER_THREADS) {
        const CtSplat p = src[i];
        if (p.r >= 0 && p.c == ch && p.y - p.r <= y1 && p.y + p.r >= y0) sh[atomicAdd(&cnt, 1)] = p;   // order-free: the max commutes
    }
    __syncthreads();
    const int n = cnt;
    float* plane = ch < s.C ? hm + ((size_t)b * s.C + ch) * s.hm_h * s.hm_w
                            : hm_hp + ((size_t)b * s.K + (ch - s.C)) * s.hm_h * s.hm_w;
    const int quads = (s.hm_w + 3) / 4;
    const bool vec = (s.hm_w & 3) == 0;
    for (int i = threadIdx.x; i < (y1 - y0 + 1) * quads; i += CT_RENDER_THREADS) {
        const int y = y0 + i / quads, x = (i % quads) * 4;
        float v[4];
        for (int j = 0; j < 4; ++j) v[j] = n ? ct_pixel(sh, n, x + j, y) : 0.f;
        float* row = plane + (size_t)y * s.hm_w;
        if (vec) {
            *(float4*)(row + x) = make_float4(v[0], v[1], v[2], v[3]);
        } else {
            for (int j = 0; j < 4 && x + j < s.hm_w; ++j) row[x + j] = v[j];
        }
    }
}

static int check_shape(int mode, int img_h, int img_w, int num_classes) {
    VD3D_REQUIRE(mode == CT_KM3D || mode == CT_MONOFLEX, "center_targets: unknown mode %d", mode);
    VD3D_REQUIRE(img_h >= CT_SCALE && img_w >= CT_SCALE && img_h <= (1 << 15) && img_w <= (1 << 15),
                 "center_targets: image size %dx%d outside [4, 32768]", img_h, img_w);
    VD3D_REQUIRE(num_classes > 0 && num_classes <= CT_MAX_CLASSES, "center_targets: %d classes outside [1, %d]", num_classes, CT_MAX_CLASSES);
    return VD3D_OK;
}

static int check_record(const CtRecord& r, int mode, int img_h, int img_w, int num_classes) {
    VD3D_REQUIRE(r.mode == mode && r.img_h == img_h && r.img_w == img_w && r.num_classes == num_classes,
                 "center_targets: record made for mode %d, %dx%d, %d classes; asked for mode %d, %dx%d, %d classes",
                 r.mode, r.img_h, r.img_w, r.num_classes, mode, img_h, img_w, num_classes);
    VD3D_REQUIRE(r.n >= 0 && r.n <= CT_MAX_OBJ, "center_targets: %d objects (max_objects = %d)", r.n, CT_MAX_OBJ);
    for (int k = 0; k < r.n; ++k)
        VD3D_REQUIRE(r.cls[k] >= 0 && r.cls[k] < num_classes, "center_targets: object %d has class %d of %d", k, r.cls[k], num_classes);
    return VD3D_OK;
}

}  // namespace vd3d

using namespace vd3d;

extern "C" int vd3d_center_targets_record_bytes(void) { return (int)sizeof(CtRecord); }

extern "C" int vd3d_center_targets_pack(void* rec, int mode, int img_h, int img_w, int num_classes, const double* P2, int n,
                                        const double* objs, const int* cls) {
    VD3D_REQUIRE(rec && P2 && (n == 0 || (objs && cls)), "center_targets_pack: null argument");
    int rc = check_shape(mode, img_h, img_w, num_classes);
    if (rc) return rc;
    VD3D_REQUIRE(n >= 0 && n <= CT_MAX_OBJ, "center_targets_pack: %d objects (max_objects = %d)", n, CT_MAX_OBJ);
    CtRecord r;
    memset(&r, 0, sizeof(r));
    for (int i = 0; i < 12; ++i) {
        VD3D_REQUIRE(isfinite(P2[i]), "center_targets_pack: P2 is not finite");
        r.P2[i] = P2[i];
    }
    VD3D_REQUIRE(P2[0] != 0.0, "center_targets_pack: P2[0, 0] == 0");
    for (int k = 0; k < n; ++k) {
        for (int f = 0; f < CT_FIELDS; ++f) {
            VD3D_REQUIRE(isfinite(objs[k * CT_FIELDS + f]), "center_targets_pack: object %d field %d is not finite", k, f);
            r.obj[k][f] = objs[k * CT_FIELDS + f];
        }
        r.cls[k] = cls[k];
    }
    r.n = n; r.mode = mode; r.img_h = img_h; r.img_w = img_w; r.num_classes = num_classes;
    rc = check_record(r, mode, img_h, img_w, num_classes);
    if (rc) return rc;
    memcpy(rec, &r, sizeof(r));
    return VD3D_OK;
}

// One image on the HOST: `outs` = CT_NOUT host pointers to that image's arrays (the three MonoFlex-only slots may be null for KM3D).
extern "C" int vd3d_center_targets_host(const void* rec, int mode, int img_h, int img_w, int num_classes, void* const* outs) {
    VD3D_REQUIRE(rec && outs, "center_targets_host: null argument");
    int rc = check_shape(mode, img_h, img_w, num_classes);
    if (rc) return rc;
    CtRecord r;
    memcpy(&r, rec, sizeof(r));
    rc = check_record(r, mode, img_h, img_w, num_classes);
    if (rc) return rc;
    const CtShape s = ct_shape(mode, img_h, img_w, num_classes);
    CtOut o;
    for (int i = 0; i < CT_NOUT; ++i) {
        o.p[i] = outs[i];
        VD3D_REQUIRE(o.p[i] || (mode == CT_KM3D && i >= O_KP_DEPTH_MASK), "center_targets_host: output %d is null", i);
    }
    CtSplat sp[CT_SPLATS];
    for (int k = 0; k < CT_MAX_OBJ; ++k) ct_object(r, s, 0, k, o, sp);
    CtSplat mine[CT_MAX_OBJ];
    for (int ch = 0; ch < s.C + s.K; ++ch) {
        int n = 0;
        for (int i = 0; i < CT_MAX_OBJ * (1 + s.K); ++i)
            if (sp[i].r >= 0 && sp[i].c == ch) mine[n++] = sp[i];
        float* plane = ch < s.C ? (float*)o.p[O_HM] + (size_t)ch * s.hm_h * s.hm_w : (float*)o.p[O_HM_HP] + (size_t)(ch - s.C) * s.hm_h * s.hm_w;
        for (int y = 0; y < s.hm_h; ++y)
            for (int x = 0; x < s.hm_w; ++x) plane[(size_t)y * s.hm_w + x] = ct_pixel(mine, n, x, y);
    }
    return VD3D_OK;
}

// Batched device form: `recs_dev` = B records (vd3d_center_targets_pack, one mode / size / class count), `outs` = a HOST array of CT_NOUT
// DEVICE pointers to the batch's [B, ...] arrays, `splats_dev` = B * vd3d_center_targets_splat_bytes() bytes of scratch.  Two launches.
extern "C" int vd3d_center_targets_splat_bytes(void) { return (int)(CT_SPLATS * sizeof(CtSplat)); }

extern "C" int vd3d_center_targets(const void* recs_dev, int B, int mode, int img_h, int img_w, int num_classes, void* const* outs,
                                   void* splats_dev, void* stream) {
    VD3D_REQUIRE(recs_dev && outs && splats_dev && B > 0 && B <= 65535, "center_targets: bad arguments (B %d)", B);
    int rc = check_shape(mode, img_h, img_w, num_classes);
    if (rc) return rc;
    const CtShape s = ct_shape(mode, img_h, img_w, num_classes);
    CtOut o;
    for (int i = 0; i < CT_NOUT; ++i) {
        o.p[i] = outs[i];
        VD3D_REQUIRE(o.p[i] || (mode == CT_KM3D && i >= O_KP_DEPTH_MASK), "center_targets: output %d is null", i);
    }
    cudaStream_t st = (cudaStream_t)stream;
    center_targets_object_kernel<<<cdiv(B, CT_OBJ_WARPS), CT_OBJ_WARPS * 32, 0, st>>>((const CtRecord*)recs_dev, B, s, o, (CtSplat*)splats_dev);
    VD3D_CHECK_LAUNCH("center_targets_object");
    dim3 grid(cdiv(s.hm_h, CT_RENDER_ROWS), s.C + s.K, B);
    center_targets_render_kernel<<<grid, CT_RENDER_THREADS, 0, st>>>((const CtSplat*)splats_dev, s, (float*)o.p[O_HM], (float*)o.p[O_HM_HP]);
    VD3D_CHECK_LAUNCH("center_targets_render");
    return VD3D_OK;
}
