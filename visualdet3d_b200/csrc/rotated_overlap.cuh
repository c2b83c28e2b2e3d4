// Overlap area of two rotated bird's-eye-view rectangles [x1, y1, x2, y2, ry] (R/lib/ops/iou3d/src/iou3d_kernel.cu:34-221, step for step
// so results agree to rounding): rotate the 4 corners of both rectangles about their centres, collect (a) the proper intersections of the
// 4 x 4 edge pairs and (b) every corner of one rectangle lying inside the other (1e-5 margin), order the points by angle about their mean,
// and take the shoelace area of the fan from the first point.  Shared by iou3d.cu and km3d_loss.cu.
#pragma once
#include <cuda_runtime.h>

namespace vd3d {

constexpr float IOU_EPS = 1e-8f;

struct P2 { float x, y; };

__device__ __forceinline__ float cross3(const P2& p1, const P2& p2, const P2& p0) {
    return (p1.x - p0.x) * (p2.y - p0.y) - (p2.x - p0.x) * (p1.y - p0.y);
}

// proper intersection of segments (p0,p1) and (q0,q1); returns false when they do not strictly cross
__device__ __forceinline__ bool seg_intersect(const P2& p1, const P2& p0, const P2& q1, const P2& q0, P2& out) {
    // bounding-box rejection (inclusive)
    bool bb = fminf(p0.x, p1.x) <= fmaxf(q0.x, q1.x) && fminf(q0.x, q1.x) <= fmaxf(p0.x, p1.x) &&
              fminf(p0.y, p1.y) <= fmaxf(q0.y, q1.y) && fminf(q0.y, q1.y) <= fmaxf(p0.y, p1.y);
    if (!bb) return false;
    float s1 = cross3(q0, p1, p0);
    float s2 = cross3(p1, q1, p0);
    float s3 = cross3(p0, q1, q0);
    float s4 = cross3(q1, p1, q0);
    if (!(s1 * s2 > 0.f && s3 * s4 > 0.f)) return false;
    float s5 = cross3(q1, p1, p0);
    if (fabsf(s5 - s1) > IOU_EPS) {
        out.x = (s5 * q0.x - s1 * q1.x) / (s5 - s1);
        out.y = (s5 * q0.y - s1 * q1.y) / (s5 - s1);
    } else {
        float a0 = p0.y - p1.y, b0 = p1.x - p0.x, c0 = p0.x * p1.y - p1.x * p0.y;
        float a1 = q0.y - q1.y, b1 = q1.x - q0.x, c1 = q0.x * q1.y - q1.x * q0.y;
        float D = a0 * b1 - a1 * b0;
        out.x = (b0 * c1 - b1 * c0) / D;
        out.y = (a1 * c0 - a0 * c1) / D;
    }
    return true;
}

__device__ __forceinline__ bool inside_box(const float* box, const P2& p) {
    const float MARGIN = 1e-5f;
    float cx = (box[0] + box[2]) / 2, cy = (box[1] + box[3]) / 2;
    float ac = cosf(-box[4]), as = sinf(-box[4]);
    float rx = (p.x - cx) * ac + (p.y - cy) * as + cx;
    float ry = -(p.x - cx) * as + (p.y - cy) * ac + cy;
    return rx > box[0] - MARGIN && rx < box[2] + MARGIN && ry > box[1] - MARGIN && ry < box[3] + MARGIN;
}

__device__ __forceinline__ void rotated_corners(const float* box, P2 (&c)[5]) {
    float x1 = box[0], y1 = box[1], x2 = box[2], y2 = box[3];
    float cx = (x1 + x2) / 2, cy = (y1 + y2) / 2;
    float ac = cosf(box[4]), as = sinf(box[4]);
    const float px[4] = {x1, x2, x2, x1}, py[4] = {y1, y1, y2, y2};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        c[k].x = (px[k] - cx) * ac + (py[k] - cy) * as + cx;
        c[k].y = -(px[k] - cx) * as + (py[k] - cy) * ac + cy;
    }
    c[4] = c[0];
}

__device__ inline float rotated_overlap(const float* a, const float* b) {
    P2 ca[5], cb[5];
    rotated_corners(a, ca);
    rotated_corners(b, cb);
    P2 pts[16];
    float sx = 0.f, sy = 0.f;
    int n = 0;
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            P2 x;
            if (seg_intersect(ca[i + 1], ca[i], cb[j + 1], cb[j], x)) { pts[n++] = x; sx += x.x; sy += x.y; }
        }
    for (int k = 0; k < 4; ++k) {
        if (inside_box(a, cb[k])) { pts[n++] = cb[k]; sx += cb[k].x; sy += cb[k].y; }
        if (inside_box(b, ca[k])) { pts[n++] = ca[k]; sx += ca[k].x; sy += ca[k].y; }
    }
    float mx = sx / n, my = sy / n;          // n == 0 -> NaN centre, never used (no points)
    // order by angle about the mean: stable exchange sort (same ordering as the reference's bubble sort with a strict '>')
    float ang[16];
    for (int i = 0; i < n; ++i) ang[i] = atan2f(pts[i].y - my, pts[i].x - mx);
    for (int j = 0; j < n - 1; ++j)
        for (int i = 0; i < n - j - 1; ++i)
            if (ang[i] > ang[i + 1]) {
                float t = ang[i]; ang[i] = ang[i + 1]; ang[i + 1] = t;
                P2 tp = pts[i]; pts[i] = pts[i + 1]; pts[i + 1] = tp;
            }
    float area = 0.f;
    for (int k = 0; k < n - 1; ++k) {
        float ax = pts[k].x - pts[0].x, ay = pts[k].y - pts[0].y;
        float bx = pts[k + 1].x - pts[0].x, by = pts[k + 1].y - pts[0].y;
        area += ax * by - ay * bx;
    }
    return fabsf(area) / 2.0f;
}

}  // namespace vd3d
