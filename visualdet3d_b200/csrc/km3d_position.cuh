// KM3D's gen_position (R/networks/utils/rtm3d_utils.py:314-455): the observation angle from the rotation bins, rot_y through the
// centre keypoint's x, and the camera-frame position as the least-squares solution of the 16 keypoint equations.  Shared by the
// detector's decode (centernet.cu) and the training loss (km3d_loss.cu), which also reads the intermediates for its backward.
#pragma once
#include <cuda_runtime.h>

namespace vd3d {

struct Km3dPosition {
    float alpha, rot_y;
    float co, si;                      // cos / sin of rot_y
    float lc, ls, wc, wsn, hh;         // l/2 cos, l/2 sin, w/2 cos, w/2 sin, h/2
    float cc[8];                       // C of corner j (rows 2j and 2j+1)
    float a2[16];                      // A's third column: the normalised keypoints (row 2j: x of corner j, row 2j+1: its y)
    float bv[16];                      // b = B - a2 * C
    double inv[3][3];                  // (A^T A)^-1
    float pos[3];                      // (pinv @ A^T).float() @ b, x shifted by -P[0,3] / P[0,0]
};

// kx / ky: the 9 keypoints at input scale (x4); dw, dh, dl: the dim channels (whl); rot: the 8 rotation channels; P: P2 [3][4].
// A row 2j = [-1, 0, nx_j], row 2j+1 = [0, -1, ny_j]; A^T A and its inverse in float64, pinv @ A^T rounded to float32 and multiplied
// by b in float32, like the reference's .double() / .float() casts.
__device__ __forceinline__ void km3d_gen_position(const float (&kx)[9], const float (&ky)[9], float dw, float dh, float dl, const float* rot,
                                                  const float* P, Km3dPosition& s) {
    const float f = P[0], pcx = P[2], pcy = P[6];
    float a1 = atanf(rot[2] / rot[3]) + (-0.5f * 3.14159265358979323846f);
    float a2 = atanf(rot[6] / rot[7]) + (0.5f * 3.14159265358979323846f);
    float sel = (rot[1] > rot[5]) ? 1.f : 0.f;
    s.alpha = a1 * sel + a2 * (1.f - sel);
    float rot_y = s.alpha + atan2f(kx[8] - pcx, f);
    const float PI = 3.14159265358979323846f;
    if (rot_y > PI) rot_y = rot_y - 2.f * PI;
    if (rot_y < -PI) rot_y = rot_y + 2.f * PI;
    s.rot_y = rot_y;
    float co = cosf(rot_y), si = sinf(rot_y);
    float lc = dl * 0.5f * co, ls = dl * 0.5f * si, wc = dw * 0.5f * co, wsn = dw * 0.5f * si, hh = dh * 0.5f;
    s.co = co; s.si = si; s.lc = lc; s.ls = ls; s.wc = wc; s.wsn = wsn; s.hh = hh;
    // rows 2j (x of corner j) and 2j+1 (y of corner j), corners 0..7
    const float Bx[8] = {-lc - wsn, -lc + wsn, -lc + wsn, lc + wsn, lc + wsn, lc - wsn, lc - wsn, -lc - wsn};
    const float By[8] = {-hh, -hh, hh, hh, -hh, -hh, hh, hh};
    const float Cc[8] = {ls - wc, ls + wc, ls + wc, -ls + wc, -ls + wc, -ls - wc, -ls - wc, ls - wc};
    double ata[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        float nx = (kx[j] - pcx) / f, ny = (ky[j] - pcy) / f;
        s.cc[j] = Cc[j];
        s.a2[2 * j] = nx; s.a2[2 * j + 1] = ny;
        s.bv[2 * j] = Bx[j] - nx * Cc[j];
        s.bv[2 * j + 1] = By[j] - ny * Cc[j];
    }
#pragma unroll
    for (int q = 0; q < 16; ++q) {
        double a0 = (q & 1) ? 0.0 : -1.0, a1d = (q & 1) ? -1.0 : 0.0, a2d = (double)s.a2[q];
        ata[0][0] += a0 * a0; ata[0][1] += a0 * a1d; ata[0][2] += a0 * a2d;
        ata[1][1] += a1d * a1d; ata[1][2] += a1d * a2d; ata[2][2] += a2d * a2d;
    }
    ata[1][0] = ata[0][1]; ata[2][0] = ata[0][2]; ata[2][1] = ata[1][2];
    // 3x3 inverse (double)
    double c00 = ata[1][1] * ata[2][2] - ata[1][2] * ata[2][1], c01 = ata[0][2] * ata[2][1] - ata[0][1] * ata[2][2], c02 = ata[0][1] * ata[1][2] - ata[0][2] * ata[1][1];
    double c10 = ata[1][2] * ata[2][0] - ata[1][0] * ata[2][2], c11 = ata[0][0] * ata[2][2] - ata[0][2] * ata[2][0], c12 = ata[0][2] * ata[1][0] - ata[0][0] * ata[1][2];
    double c20 = ata[1][0] * ata[2][1] - ata[1][1] * ata[2][0], c21 = ata[0][1] * ata[2][0] - ata[0][0] * ata[2][1], c22 = ata[0][0] * ata[1][1] - ata[0][1] * ata[1][0];
    double det = ata[0][0] * c00 + ata[0][1] * c10 + ata[0][2] * c20;
    const double cof[3][3] = {{c00, c01, c02}, {c10, c11, c12}, {c20, c21, c22}};
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) s.inv[i][j] = cof[i][j] / det;
    float pos[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int q = 0; q < 16; ++q) {
        double a0 = (q & 1) ? 0.0 : -1.0, a1d = (q & 1) ? -1.0 : 0.0, a2d = (double)s.a2[q];
#pragma unroll
        for (int rI = 0; rI < 3; ++rI) {
            float pq = (float)(s.inv[rI][0] * a0 + s.inv[rI][1] * a1d + s.inv[rI][2] * a2d);     // (pinv @ A^T).float()
            pos[rI] = fmaf(pq, s.bv[q], pos[rI]);
        }
    }
    pos[0] -= P[3] / P[0];
    s.pos[0] = pos[0]; s.pos[1] = pos[1]; s.pos[2] = pos[2];
}

}  // namespace vd3d
