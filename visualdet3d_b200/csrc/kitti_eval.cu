// KITTI object evaluator (bbox / BEV / 3-D AP and AOS) for sm_90a: the arithmetic of the reference's numba evaluator
// (R/evaluator/kitti/eval.py, rotate_iou.py), decomposed per image instead of per 50-image "part".
//
// Data (all device, float64 as parsed): ground truth [n_gt][KE_GT_COLS], detections [n_dt][KE_DT_COLS] (the same columns + score),
// CSR offsets offs[4][n_img+1] = ground truth, detections, [dt x gt] overlap blocks, 32-bit detection-flag words.
// Configuration index cfg = ((metric * n_cls + class) * 3 + difficulty) * n_mo + row, over the n_mo min-overlap rows: the reference's
// precision[class][difficulty][row][41] per metric, flattened.  The official evaluation has n_mo = 2, the COCO-style one 10.
//
// Compiled with -fmad=false: the bbox overlaps and all float64 statistics then round every product and sum separately, like numba.
#include "common.cuh"
#include <cub/device/device_segmented_radix_sort.cuh>
#include <math_constants.h>

using vd3d::cdiv;

namespace {

constexpr int kGtCols = 15;       // bbox x1 y1 x2 y2, alpha, l h w, x y z, ry, truncated, occluded, class code
constexpr int kDtCols = 16;       // the same + score
constexpr int kPts = 41;          // N_SAMPLE_PTS
constexpr int kMaxInter = 24;     // 8 corners inside the other box + 16 edge crossings
constexpr double kNoDetection = -10000000.0;
enum { C_X1 = 0, C_Y1, C_X2, C_Y2, C_ALPHA, C_L, C_H, C_W, C_X, C_Y, C_Z, C_RY, C_TRUNC, C_OCC, C_CODE, C_SCORE };
constexpr int kDontCare = -2;     // class code of a ground-truth row named exactly "DontCare"

// ---- rotated IoU in float32 (rotate_iou.py: devRotateIoUEval and helpers, same expression order) ---------------------------
__device__ __forceinline__ float tri_area(float ax, float ay, float bx, float by, float cx, float cy) {
    return ((ax - cx) * (by - cy) - (ay - cy) * (bx - cx)) / 2.0f;
}

// corners clockwise, rotated clockwise by the angle; cos / sin are taken in double and rounded, as the reference's math.cos does
__device__ void rbox_corners(const float* b, float* c) {
    const float a_cos = (float)cos((double)b[4]), a_sin = (float)sin((double)b[4]);
    const float hx = -b[2] / 2.0f, hy = -b[3] / 2.0f, px = b[2] / 2.0f, py = b[3] / 2.0f;
    const float cx[4] = {hx, hx, px, px}, cy[4] = {hy, py, py, hy};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        c[2 * i] = a_cos * cx[i] + a_sin * cy[i] + b[0];
        c[2 * i + 1] = -a_sin * cx[i] + a_cos * cy[i] + b[1];
    }
}

__device__ __forceinline__ bool point_in_quad(float x, float y, const float* c) {
    const float ab0 = c[2] - c[0], ab1 = c[3] - c[1], ad0 = c[6] - c[0], ad1 = c[7] - c[1];
    const float ap0 = x - c[0], ap1 = y - c[1];
    const float abab = ab0 * ab0 + ab1 * ab1, abap = ab0 * ap0 + ab1 * ap1;
    const float adad = ad0 * ad0 + ad1 * ad1, adap = ad0 * ap0 + ad1 * ap1;
    return abab >= abap && abap >= 0 && adad >= adap && adap >= 0;
}

// line_segment_intersection (the strict-comparison form, not _v1)
__device__ bool seg_intersect(const float* p1, const float* p2, int i, int j, float* out) {
    const float A0 = p1[2 * i], A1 = p1[2 * i + 1], B0 = p1[2 * ((i + 1) % 4)], B1 = p1[2 * ((i + 1) % 4) + 1];
    const float C0 = p2[2 * j], C1 = p2[2 * j + 1], D0 = p2[2 * ((j + 1) % 4)], D1 = p2[2 * ((j + 1) % 4) + 1];
    const float BA0 = B0 - A0, BA1 = B1 - A1, DA0 = D0 - A0, CA0 = C0 - A0, DA1 = D1 - A1, CA1 = C1 - A1;
    const bool acd = DA1 * CA0 > CA1 * DA0;
    const bool bcd = (D1 - B1) * (C0 - B0) > (C1 - B1) * (D0 - B0);
    if (acd != bcd) {
        const bool abc = CA1 * BA0 > BA1 * CA0;
        const bool abd = DA1 * BA0 > BA1 * DA0;
        if (abc != abd) {
            const float DC0 = D0 - C0, DC1 = D1 - C1;
            const float ABBA = A0 * B1 - B0 * A1, CDDC = C0 * D1 - D0 * C1;
            const float DH = BA1 * DC0 - BA0 * DC1;
            const float Dx = ABBA * DC0 - BA0 * CDDC, Dy = ABBA * DC1 - BA1 * CDDC;
            out[0] = Dx / DH;
            out[1] = Dy / DH;
            return true;
        }
    }
    return false;
}

// intersection area of two rotated boxes (x, y, dx, dy, angle): inter() of the reference, with room for all 24 candidate points
__device__ float rbox_inter(const float* b1, const float* b2) {
    float c1[8], c2[8], p[2 * kMaxInter], vs[kMaxInter];
    rbox_corners(b1, c1);
    rbox_corners(b2, c2);
    int n = 0;
    for (int i = 0; i < 4; ++i) {
        if (point_in_quad(c1[2 * i], c1[2 * i + 1], c2)) { p[2 * n] = c1[2 * i]; p[2 * n + 1] = c1[2 * i + 1]; ++n; }
        if (point_in_quad(c2[2 * i], c2[2 * i + 1], c1)) { p[2 * n] = c2[2 * i]; p[2 * n + 1] = c2[2 * i + 1]; ++n; }
    }
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            float t[2];
            if (seg_intersect(c1, c2, i, j, t)) { p[2 * n] = t[0]; p[2 * n + 1] = t[1]; ++n; }
        }
    if (n > 0) {   // sort_vertex_in_convex_polygon: insertion sort on the pseudo-angle around the centroid
        float cx = 0.0f, cy = 0.0f;
        for (int i = 0; i < n; ++i) { cx += p[2 * i]; cy += p[2 * i + 1]; }
        cx /= (float)n;
        cy /= (float)n;
        for (int i = 0; i < n; ++i) {
            float v0 = p[2 * i] - cx, v1 = p[2 * i + 1] - cy;
            const float d = sqrtf(v0 * v0 + v1 * v1);
            v0 = v0 / d;
            v1 = v1 / d;
            if (v1 < 0) v0 = -2 - v0;
            vs[i] = v0;
        }
        for (int i = 1; i < n; ++i) {
            if (vs[i - 1] > vs[i]) {
                const float temp = vs[i], tx = p[2 * i], ty = p[2 * i + 1];
                int j = i;
                while (j > 0 && vs[j - 1] > temp) {
                    vs[j] = vs[j - 1];
                    p[2 * j] = p[2 * j - 2];
                    p[2 * j + 1] = p[2 * j - 1];
                    --j;
                }
                vs[j] = temp;
                p[2 * j] = tx;
                p[2 * j + 1] = ty;
            }
        }
    }
    float area = 0.0f;   // fan triangulation from the first vertex
    for (int i = 0; i < n - 2; ++i)
        area += fabsf(tri_area(p[0], p[1], p[2 * i + 2], p[2 * i + 3], p[2 * i + 4], p[2 * i + 5]));
    return area;
}

// devRotateIoUEval(rbox1, rbox2, criterion): not symmetric in float32, so callers keep the reference's (query box, box) order
__device__ float rotate_iou_eval(const float* r1, const float* r2, int criterion) {
    const float area1 = r1[2] * r1[3], area2 = r2[2] * r2[3];
    const float inter = rbox_inter(r1, r2);
    if (criterion == -1) return inter / (area1 + area2 - inter);
    if (criterion == 0) return inter / area1;
    if (criterion == 1) return inter / area2;
    return inter;
}

__global__ void rotate_iou_kernel(const float* __restrict__ boxes, int N, const float* __restrict__ qboxes, int K, int criterion,
                                  float* __restrict__ iou) {
    const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (t >= (long long)N * K) return;
    const int n = (int)(t / K), k = (int)(t % K);
    float b[5], q[5];
    for (int c = 0; c < 5; ++c) { b[c] = boxes[5 * n + c]; q[c] = qboxes[5 * k + c]; }
    iou[t] = rotate_iou_eval(q, b, criterion);
}

// ---- bbox overlap: image_box_overlap(boxes, query_boxes, criterion) for one pair, float64 in the reference's order --------------
__device__ __forceinline__ double box_overlap(const double* b, const double* q, int criterion) {
    const double qa = (q[2] - q[0]) * (q[3] - q[1]);
    const double iw = fmin(b[2], q[2]) - fmax(b[0], q[0]);
    if (iw > 0) {
        const double ih = fmin(b[3], q[3]) - fmax(b[1], q[1]);
        if (ih > 0) {
            double ua;
            if (criterion == -1) ua = (b[2] - b[0]) * (b[3] - b[1]) + qa - iw * ih;
            else if (criterion == 0) ua = (b[2] - b[0]) * (b[3] - b[1]);
            else if (criterion == 1) ua = qa;
            else ua = 1.0;
            return iw * ih / ua;
        }
    }
    return 0.0;
}

__device__ __forceinline__ int find_image(const long long* off, int n_img, long long x) {   // largest i with off[i] <= x
    int lo = 0, hi = n_img;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (off[mid] <= x) lo = mid; else hi = mid;
    }
    return lo;
}

struct EvalArgs {
    const double* gt;
    const double* dt;
    const long long* gt_off;
    const long long* dt_off;
    const long long* ov_off;
    const long long* word_off;
    int n_img, n_cls, n_mo;
    long long n_gt, n_dt, n_pairs, n_words;
    const int* classes;           // [n_cls] class indices of the reference's CLASS_NAMES
    const double* min_overlaps;   // [n_mo][3][n_cls]
    int compute_aos;
    double* overlaps;             // [3][n_pairs]: per image [dt][gt] row-major
    signed char* ign_gt;          // [n_cls][3][n_gt]
    signed char* ign_dt;          // [n_cls][3][n_dt]
    int* n_valid;                 // [n_cls][3]
    unsigned* flags1;             // [n_cfg][n_words]
    double* tp_scores;            // [n_cfg][n_gt]
    double* tp_sorted;            // [n_cfg][n_gt]
    int* n_tp;                    // [n_cfg]
    double* thresholds;           // [n_cfg][41]
    int* n_thresh;                // [n_cfg]
    unsigned* flags2;             // [n_cfg][41][n_words]
    int* counts;                  // [n_cfg][41][3] tp, fp, fn
    double* sims;                 // [3 n_mo n_cls][41][n_img]
    double* precision;            // [n_cfg][41]
    double* orientation;          // [3 n_mo n_cls][41]
};

// ---- overlaps of the three metrics, one thread per (metric, dt, gt) pair of one image ------------------------------------------
__global__ void overlap_kernel(EvalArgs a) {
    const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    const int metric = blockIdx.y;
    if (t >= a.n_pairs) return;
    const int img = find_image(a.ov_off, a.n_img, t);
    const long long ng = a.gt_off[img + 1] - a.gt_off[img];
    const long long local = t - a.ov_off[img];
    const double* d = a.dt + (a.dt_off[img] + local / ng) * kDtCols;
    const double* g = a.gt + (a.gt_off[img] + local % ng) * kGtCols;
    double ov;
    if (metric == 0) {
        ov = box_overlap(d, g, -1);                  // boxes = detections, query_boxes = ground truth
    } else {
        const float gb[5] = {(float)g[C_X], (float)g[C_Z], (float)g[C_L], (float)g[C_W], (float)g[C_RY]};
        const float db[5] = {(float)d[C_X], (float)d[C_Z], (float)d[C_L], (float)d[C_W], (float)d[C_RY]};
        if (metric == 1) {
            ov = (double)rotate_iou_eval(gb, db, -1);
        } else {   // d3_box_overlap_kernel, z_axis = 1, z_center = 1.0, criterion -1; the result is stored as float32 like its rinc buffer
            const float rinc = rotate_iou_eval(gb, db, 2);
            float r = rinc;
            if (rinc > 0) {
                const double min_z = fmin(d[C_Y] + d[C_H] * (1 - 1.0), g[C_Y] + g[C_H] * (1 - 1.0));
                const double max_z = fmax(d[C_Y] - d[C_H] * 1.0, g[C_Y] - g[C_H] * 1.0);
                const double iw = min_z - max_z;
                if (iw > 0) {
                    const double area1 = d[C_L] * d[C_H] * d[C_W], area2 = g[C_L] * g[C_H] * g[C_W];
                    const double inc = iw * (double)rinc;
                    r = (float)(inc / (area1 + area2 - inc));
                } else {
                    r = 0.0f;
                }
            }
            ov = (double)r;
        }
    }
    a.overlaps[metric * a.n_pairs + t] = ov;
}

// ---- clean_data: per-box ignore flags for every (class, difficulty) -----------------------------------------------------------
__constant__ double kMinHeight[3] = {40, 25, 25};
__constant__ int kMaxOcclusion[3] = {0, 1, 2};
__constant__ double kMaxTruncation[3] = {0.15, 0.3, 0.5};

__device__ __forceinline__ int canonical_class(int c) { return c == 5 ? 0 : c; }   // CLASS_NAMES[5] is 'car' again

__global__ void clean_kernel(EvalArgs a) {
    const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    const int cd = blockIdx.y, c = cd / 3, diff = cd % 3;
    const int cls = canonical_class(a.classes[c]);
    if (t < a.n_gt) {
        const double* g = a.gt + t * kGtCols;
        const int code = (int)g[C_CODE];
        const double height = g[C_Y2] - g[C_Y1];
        int valid_class = -1;
        if (code == cls) valid_class = 1;
        else if (cls == 1 && code == 4) valid_class = 0;      // Person_sitting next to Pedestrian
        else if (cls == 0 && code == 3) valid_class = 0;      // Van next to Car
        const bool ignore = g[C_OCC] > kMaxOcclusion[diff] || g[C_TRUNC] > kMaxTruncation[diff] || height <= kMinHeight[diff];
        signed char f;
        if (valid_class == 1 && !ignore) { f = 0; atomicAdd(a.n_valid + cd, 1); }
        else if (valid_class == 0 || (ignore && valid_class == 1)) f = 1;
        else f = -1;
        a.ign_gt[cd * a.n_gt + t] = f;
    } else if (t < a.n_gt + a.n_dt) {
        const long long i = t - a.n_gt;
        const double* d = a.dt + i * kDtCols;
        const double height = fabs(d[C_Y2] - d[C_Y1]);
        signed char f;
        if (height < kMinHeight[diff]) f = 1;
        else if ((int)d[C_CODE] == cls) f = 0;
        else f = -1;
        a.ign_dt[cd * a.n_dt + i] = f;
    }
}

// ---- compute_statistics_jit for one (configuration, image, threshold) --------------------------------------------------------
struct Stats {
    int tp, fp, fn;
    double similarity;
};

__device__ __forceinline__ bool flag_get(const unsigned* w, int j) { return (w[j >> 5] >> (j & 31)) & 1u; }
__device__ __forceinline__ void flag_set(unsigned* w, int j) { w[j >> 5] |= 1u << (j & 31); }

// compute_fp == false: collects the scores of true positives into `tp_out`; compute_fp == true: counts at `thresh`
template <bool kComputeFp>
__device__ Stats compute_statistics(const EvalArgs& a, int metric, int cd, int img, double min_overlap, double thresh, bool compute_aos,
                                    unsigned* assigned, double* tp_out) {
    const long long g0 = a.gt_off[img], d0 = a.dt_off[img];
    const int ng = (int)(a.gt_off[img + 1] - g0), nd = (int)(a.dt_off[img + 1] - d0);
    const double* ov = a.overlaps + metric * a.n_pairs + a.ov_off[img];
    const signed char* ig = a.ign_gt + cd * a.n_gt + g0;
    const signed char* idt = a.ign_dt + cd * a.n_dt + d0;
    const double* dt = a.dt + d0 * kDtCols;
    const double* gt = a.gt + g0 * kGtCols;
    for (int w = 0; w < (nd + 31) / 32; ++w) assigned[w] = 0u;
    auto below = [&](int j) { return kComputeFp && dt[j * kDtCols + C_SCORE] < thresh; };   // ignored_threshold
    Stats s = {0, 0, 0, 0.0};
    double sim_sum = 0.0;
    for (int i = 0; i < ng; ++i) {
        if (ig[i] == -1) continue;
        int det_idx = -1;
        double valid_detection = kNoDetection, max_overlap = 0;
        bool assigned_ignored_det = false;
        for (int j = 0; j < nd; ++j) {
            if (idt[j] == -1 || flag_get(assigned, j) || below(j)) continue;
            const double overlap = ov[(long long)j * ng + i];
            const double dt_score = dt[j * kDtCols + C_SCORE];
            if (!kComputeFp && overlap > min_overlap && dt_score > valid_detection) {
                det_idx = j;
                valid_detection = dt_score;
            } else if (kComputeFp && overlap > min_overlap && (overlap > max_overlap || assigned_ignored_det) && idt[j] == 0) {
                max_overlap = overlap;
                det_idx = j;
                valid_detection = 1;
                assigned_ignored_det = false;
            } else if (kComputeFp && overlap > min_overlap && valid_detection == kNoDetection && idt[j] == 1) {
                det_idx = j;
                valid_detection = 1;
                assigned_ignored_det = true;
            }
        }
        if (valid_detection == kNoDetection && ig[i] == 0) {
            s.fn += 1;
        } else if (valid_detection != kNoDetection && (ig[i] == 1 || idt[det_idx] == 1)) {
            flag_set(assigned, det_idx);
        } else if (valid_detection != kNoDetection) {
            if (!kComputeFp) tp_out[s.tp] = dt[det_idx * kDtCols + C_SCORE];
            s.tp += 1;
            if (compute_aos) {   // the reference sums (1 + cos(delta)) / 2 over the true positives in this order
                const double delta = gt[i * kGtCols + C_ALPHA] - dt[det_idx * kDtCols + C_ALPHA];
                sim_sum += (1.0 + cos(delta)) / 2.0;
            }
            flag_set(assigned, det_idx);
        }
    }
    if (kComputeFp) {
        for (int j = 0; j < nd; ++j)
            if (!(flag_get(assigned, j) || idt[j] == -1 || idt[j] == 1 || below(j))) s.fp += 1;
        int nstuff = 0;
        if (metric == 0) {   // detections covered by a DontCare region (criterion 0: the detection's own area) are not false positives
            for (int i = 0; i < ng; ++i) {
                if ((int)gt[i * kGtCols + C_CODE] != kDontCare) continue;
                for (int j = 0; j < nd; ++j) {
                    if (flag_get(assigned, j) || idt[j] == -1 || idt[j] == 1 || below(j)) continue;
                    if (box_overlap(dt + j * kDtCols, gt + i * kGtCols, 0) > min_overlap) {
                        flag_set(assigned, j);
                        nstuff += 1;
                    }
                }
            }
        }
        s.fp -= nstuff;
        if (compute_aos) s.similarity = (s.tp > 0 || s.fp > 0) ? sim_sum : -1.0;
    }
    return s;
}

__device__ __forceinline__ void decode_cfg(const EvalArgs& a, int cfg, int& metric, int& cd, double& min_overlap) {
    const int k = cfg % a.n_mo;
    cd = (cfg / a.n_mo) % (a.n_cls * 3);
    metric = cfg / (a.n_mo * a.n_cls * 3);
    min_overlap = a.min_overlaps[(k * 3 + metric) * a.n_cls + cd / 3];
}

// pass 1: one thread per (configuration, image); true-positive scores go to the image's ground-truth slots, the rest are -inf
__global__ void pass1_kernel(EvalArgs a, int n_cfg) {
    const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (t >= (long long)n_cfg * a.n_img) return;
    const int cfg = (int)(t / a.n_img), img = (int)(t % a.n_img);
    int metric, cd;
    double min_overlap;
    decode_cfg(a, cfg, metric, cd, min_overlap);
    double* out = a.tp_scores + cfg * a.n_gt + a.gt_off[img];
    const Stats s = compute_statistics<false>(a, metric, cd, img, min_overlap, 0.0, false, a.flags1 + cfg * a.n_words + a.word_off[img], out);
    const int ng = (int)(a.gt_off[img + 1] - a.gt_off[img]);
    for (int i = s.tp; i < ng; ++i) out[i] = -CUDART_INF;
    if (s.tp) atomicAdd(a.n_tp + cfg, s.tp);
}

// get_thresholds: one sequential scan per configuration over its scores sorted descending
__global__ void thresholds_kernel(EvalArgs a, int n_cfg) {
    const int cfg = blockIdx.x * blockDim.x + threadIdx.x;
    if (cfg >= n_cfg) return;
    const int n = a.n_tp[cfg];
    const int num_gt = a.n_valid[(cfg / a.n_mo) % (a.n_cls * 3)];
    const double* sc = a.tp_sorted + cfg * a.n_gt;
    double* thr = a.thresholds + cfg * kPts;
    double current_recall = 0;
    int nt = 0;
    for (int i = 0; i < n; ++i) {
        const double l_recall = (double)(i + 1) / (double)num_gt;
        const double r_recall = i < n - 1 ? (double)(i + 2) / (double)num_gt : l_recall;
        if ((r_recall - current_recall) < (current_recall - l_recall) && i < n - 1) continue;
        if (nt < kPts) thr[nt] = sc[i];
        ++nt;
        current_recall += 1 / (kPts - 1.0);
    }
    for (int i = nt; i < kPts; ++i) thr[i] = 0.0;
    a.n_thresh[cfg] = nt;
}

// pass 2 (fused_compute_statistics): one thread per (configuration, image, threshold); counts are exact integer sums, the AOS
// similarity is stored per image and summed in image order by finalize_kernel
__global__ void pass2_kernel(EvalArgs a, int n_cfg) {
    const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (t >= (long long)n_cfg * a.n_img * kPts) return;
    const int ti = (int)(t % kPts);
    const long long ci = t / kPts;
    const int cfg = (int)(ci / a.n_img), img = (int)(ci % a.n_img);
    if (ti >= min(a.n_thresh[cfg], kPts)) return;
    int metric, cd;
    double min_overlap;
    decode_cfg(a, cfg, metric, cd, min_overlap);
    const bool aos = a.compute_aos && metric == 0;
    unsigned* flags = a.flags2 + ((long long)cfg * kPts + ti) * a.n_words + a.word_off[img];
    const Stats s = compute_statistics<true>(a, metric, cd, img, min_overlap, a.thresholds[cfg * kPts + ti], aos, flags, nullptr);
    int* c = a.counts + (cfg * kPts + ti) * 3;
    if (s.tp) atomicAdd(c + 0, s.tp);
    if (s.fp) atomicAdd(c + 1, s.fp);
    if (s.fn) atomicAdd(c + 2, s.fn);
    if (aos) a.sims[((long long)cfg * kPts + ti) * a.n_img + img] = s.similarity;   // metric-0 configurations come first
}

__device__ __forceinline__ double nan_max(double x, double y) { return (isnan(x) || isnan(y)) ? CUDART_NAN : fmax(x, y); }

// precision = tp / (tp + fp) and aos = similarity / (tp + fp) per threshold, then the running max from the right (np.max propagates NaN)
__global__ void finalize_kernel(EvalArgs a) {
    const int cfg = blockIdx.x, ti = threadIdx.x;
    __shared__ double prec[kPts], orient[kPts];
    int metric, cd;
    double mo;
    decode_cfg(a, cfg, metric, cd, mo);
    const bool aos = a.compute_aos && metric == 0;
    if (ti < kPts) {
        double p = 0.0, o = 0.0;
        if (ti < min(a.n_thresh[cfg], kPts)) {
            const int* c = a.counts + (cfg * kPts + ti) * 3;
            const double tp = (double)c[0], fp = (double)c[1];
            p = tp / (tp + fp);
            if (aos) {
                double sim = 0.0;
                const double* s = a.sims + ((long long)cfg * kPts + ti) * a.n_img;
                for (int i = 0; i < a.n_img; ++i)
                    if (s[i] != -1) sim += s[i];
                o = sim / (tp + fp);
            }
        }
        prec[ti] = p;
        orient[ti] = o;
    }
    __syncthreads();
    if (ti == 0) {
        const int nt = min(a.n_thresh[cfg], kPts);
        for (int i = nt - 1; i >= 0; --i) {
            prec[i] = nan_max(prec[i], prec[i + 1 < kPts ? i + 1 : i]);
            orient[i] = nan_max(orient[i], orient[i + 1 < kPts ? i + 1 : i]);
        }
    }
    __syncthreads();
    if (ti < kPts) {
        a.precision[cfg * kPts + ti] = prec[ti];
        if (metric == 0) a.orientation[cfg * kPts + ti] = orient[ti];
    }
}

__global__ void fill_segments_kernel(int* seg, int n_cfg, long long n_gt) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= n_cfg) seg[i] = (int)(i * n_gt);
}

// ---- workspace layout ---------------------------------------------------------------------------------------------------------
struct Layout {
    size_t ign_gt, ign_dt, n_valid, flags1, tp_scores, tp_sorted, n_tp, n_thresh, flags2, counts, sims, seg, cub, total;
    size_t cub_bytes;
};

size_t align_up(size_t x) { return (x + 255) & ~size_t(255); }

int make_layout(int n_img, long long n_gt, long long n_dt, long long n_words, int n_cls, int n_mo, Layout& L) {
    if ((long long)n_mo * n_cls > 0x7fffffffLL / (9 * kPts * 3)) return VD3D_EINVAL;   // the kernels index counts [n_cfg][41][3] with int
    const long long n_cfg = 9LL * n_mo * n_cls;
    size_t o = 0;
    auto take = [&](size_t bytes) { const size_t at = o; o = align_up(o + bytes); return at; };
    L.ign_gt = take(n_cls * 3 * n_gt);
    L.ign_dt = take(n_cls * 3 * n_dt);
    L.n_valid = take(n_cls * 3 * sizeof(int));
    L.flags1 = take(n_cfg * n_words * sizeof(unsigned));
    L.tp_scores = take(n_cfg * n_gt * sizeof(double));
    L.tp_sorted = take(n_cfg * n_gt * sizeof(double));
    L.n_tp = take(n_cfg * sizeof(int));
    L.n_thresh = take(n_cfg * sizeof(int));
    L.flags2 = take(n_cfg * kPts * n_words * sizeof(unsigned));
    L.counts = take(n_cfg * kPts * 3 * sizeof(int));
    L.sims = take(3LL * n_mo * n_cls * kPts * n_img * sizeof(double));
    L.seg = take((n_cfg + 1) * sizeof(int));
    L.cub_bytes = 0;
    if (n_cfg * n_gt > 0) {
        if (n_cfg * n_gt > 0x7fffffffLL) return VD3D_EINVAL;
        cudaError_t e = cub::DeviceSegmentedRadixSort::SortKeysDescending(nullptr, L.cub_bytes, (const double*)nullptr, (double*)nullptr,
                                                                          (int)(n_cfg * n_gt), (int)n_cfg, (const int*)nullptr,
                                                                          (const int*)nullptr + 1);
        if (e != cudaSuccess) return VD3D_ECUDA;
    }
    L.cub = take(L.cub_bytes);
    L.total = o;
    return VD3D_OK;
}

}  // namespace

extern "C" int vd3d_kitti_rotate_iou(const float* boxes, int N, const float* qboxes, int K, int criterion, float* iou, void* stream) {
    VD3D_REQUIRE(N >= 0 && K >= 0 && (N == 0 || boxes) && (K == 0 || qboxes) && (N == 0 || K == 0 || iou), "kitti_rotate_iou: bad args");
    VD3D_REQUIRE(criterion >= -1 && criterion <= 2, "kitti_rotate_iou: criterion must be -1, 0, 1 or 2");
    const long long total = (long long)N * K;
    if (total == 0) return VD3D_OK;
    rotate_iou_kernel<<<cdiv(total, 128), 128, 0, (cudaStream_t)stream>>>(boxes, N, qboxes, K, criterion, iou);
    VD3D_CHECK_LAUNCH("kitti_rotate_iou");
    return VD3D_OK;
}

extern "C" long long vd3d_kitti_eval_workspace_bytes(int n_img, long long n_gt, long long n_dt, long long n_words, int n_cls, int n_mo) {
    if (n_img < 0 || n_gt < 0 || n_dt < 0 || n_words < 0 || n_cls <= 0 || n_mo <= 0) {
        vd3d::set_error("kitti_eval_workspace_bytes: bad args");
        return VD3D_EINVAL;
    }
    Layout L;
    const int rc = make_layout(n_img, n_gt, n_dt, n_words, n_cls, n_mo, L);
    if (rc != VD3D_OK) {
        vd3d::set_error("kitti_eval_workspace_bytes: %s", rc == VD3D_EINVAL ? "too many configurations or scores for one segmented sort"
                                                                           : "cub query failed");
        return rc;
    }
    return (long long)L.total;
}

extern "C" int vd3d_kitti_eval(const double* gt, const double* dt, const long long* offs, int n_img, long long n_gt, long long n_dt,
                               long long n_pairs, long long n_words, const int* classes, int n_cls, const double* min_overlaps, int n_mo,
                               int compute_aos,
                               double* overlaps, double* precision, double* orientation, double* thresholds, int* n_thresh,
                               void* workspace, long long workspace_bytes, void* stream) {
    VD3D_REQUIRE(n_img > 0 && n_cls > 0 && n_mo > 0 && n_gt >= 0 && n_dt >= 0 && n_pairs >= 0 && n_words >= 0, "kitti_eval: bad sizes");
    VD3D_REQUIRE(offs && classes && min_overlaps && precision && orientation && thresholds && n_thresh && workspace,
                 "kitti_eval: null pointer");
    VD3D_REQUIRE((n_gt == 0 || gt) && (n_dt == 0 || dt) && (n_pairs == 0 || overlaps), "kitti_eval: null box or overlap pointer");
    Layout L;
    VD3D_REQUIRE(make_layout(n_img, n_gt, n_dt, n_words, n_cls, n_mo, L) == VD3D_OK, "kitti_eval: workspace layout failed");
    VD3D_REQUIRE((size_t)workspace_bytes >= L.total, "kitti_eval: workspace of %lld bytes, %zu needed", workspace_bytes, L.total);
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    const int n_cfg = 9 * n_mo * n_cls;   // make_layout bounded n_cfg * 41 * 3 by INT_MAX
    EvalArgs a;
    a.gt = gt; a.dt = dt;
    a.gt_off = offs; a.dt_off = offs + (n_img + 1); a.ov_off = offs + 2 * (n_img + 1); a.word_off = offs + 3 * (n_img + 1);
    a.n_img = n_img; a.n_cls = n_cls; a.n_mo = n_mo; a.n_gt = n_gt; a.n_dt = n_dt; a.n_pairs = n_pairs; a.n_words = n_words;
    a.classes = classes; a.min_overlaps = min_overlaps; a.compute_aos = compute_aos;
    a.overlaps = overlaps;
    a.ign_gt = (signed char*)(ws + L.ign_gt); a.ign_dt = (signed char*)(ws + L.ign_dt); a.n_valid = (int*)(ws + L.n_valid);
    a.flags1 = (unsigned*)(ws + L.flags1); a.tp_scores = (double*)(ws + L.tp_scores); a.tp_sorted = (double*)(ws + L.tp_sorted);
    a.n_tp = (int*)(ws + L.n_tp); a.thresholds = thresholds; a.n_thresh = n_thresh; a.flags2 = (unsigned*)(ws + L.flags2);
    a.counts = (int*)(ws + L.counts); a.sims = (double*)(ws + L.sims); a.precision = precision; a.orientation = orientation;

    VD3D_CUDA(cudaMemsetAsync(a.n_valid, 0, n_cls * 3 * sizeof(int), st));
    VD3D_CUDA(cudaMemsetAsync(a.n_tp, 0, n_cfg * sizeof(int), st));
    VD3D_CUDA(cudaMemsetAsync(a.counts, 0, (size_t)n_cfg * kPts * 3 * sizeof(int), st));
    if (n_pairs > 0) {
        overlap_kernel<<<dim3(cdiv(n_pairs, 128), 3), 128, 0, st>>>(a);
        VD3D_CHECK_LAUNCH("kitti_eval overlaps");
    }
    if (n_gt + n_dt > 0) {
        clean_kernel<<<dim3(cdiv(n_gt + n_dt, 128), n_cls * 3), 128, 0, st>>>(a);
        VD3D_CHECK_LAUNCH("kitti_eval clean_data");
    }
    pass1_kernel<<<cdiv((long long)n_cfg * n_img, 128), 128, 0, st>>>(a, n_cfg);
    VD3D_CHECK_LAUNCH("kitti_eval pass 1");
    if (n_gt > 0) {
        int* seg = (int*)(ws + L.seg);
        fill_segments_kernel<<<cdiv(n_cfg + 1, 128), 128, 0, st>>>(seg, n_cfg, n_gt);
        VD3D_CHECK_LAUNCH("kitti_eval segments");
        size_t cub_bytes = L.cub_bytes;
        VD3D_CUDA(cub::DeviceSegmentedRadixSort::SortKeysDescending(ws + L.cub, cub_bytes, a.tp_scores, a.tp_sorted, (int)(n_cfg * n_gt), n_cfg,
                                                                    seg, seg + 1, 0, sizeof(double) * 8, st));
        vd3d::count_launch();
    }
    thresholds_kernel<<<cdiv(n_cfg, 64), 64, 0, st>>>(a, n_cfg);
    VD3D_CHECK_LAUNCH("kitti_eval thresholds");
    pass2_kernel<<<cdiv((long long)n_cfg * n_img * kPts, 128), 128, 0, st>>>(a, n_cfg);
    VD3D_CHECK_LAUNCH("kitti_eval pass 2");
    finalize_kernel<<<n_cfg, 64, 0, st>>>(a);
    VD3D_CHECK_LAUNCH("kitti_eval precision");
    return VD3D_OK;
}
