// Rotated-box geometry shared by the BEV NMS kernels (bev_nms.cu, bev_nms_group.cu): the rotated IoU of detectron2's
// box_iou_rotated_utils.h, pytorch3d's quaternion <-> matrix conversions and the decoded box -> global frame -> BEV
// top-surface rectangle of postprocessing.py / boxes3d.py / bev_nms.py.  Internal linkage: every translation unit that
// includes it gets its own copy, so the kernels inline them as before.
#pragma once
#include "detect.cuh"

#include <math.h>

namespace dd3d {

namespace {

struct P2 {
    float x, y;
};

constexpr int kClipMax = 20;  // Sutherland-Hodgman output bound from a quadrilateral: 4 -> 6 -> 9 -> 13 -> 19 vertices

// One Sutherland-Hodgman step against the axis-aligned half-plane sgn * (axis ? y : x) <= lim.  A crossing point is put
// exactly on the line, and it lies between the two vertices of its edge, so a vertex that rounding places on the wrong
// side of a line it (nearly) lies on moves the area by no more than that rounding: parallel and collinear edges need no
// special case.  Returns the output count (<= n + n / 2: one extra vertex per outside -> inside transition).
__device__ int clip_half_plane(const P2* in, int n, P2* out, int axis, float sgn, float lim) {
    int m = 0;
    if (n == 0) return 0;
    P2 prev = in[n - 1];
    float dp = lim - sgn * (axis ? prev.y : prev.x);
    for (int i = 0; i < n; ++i) {
        const P2 cur = in[i];
        const float dc = lim - sgn * (axis ? cur.y : cur.x);
        if ((dc >= 0.f) != (dp >= 0.f)) {
            const float t = dp / (dp - dc);  // in [0, 1]: dp and dc have opposite signs
            const float o = axis ? prev.x + t * (cur.x - prev.x) : prev.y + t * (cur.y - prev.y);
            out[m++] = axis ? P2{o, sgn * lim} : P2{sgn * lim, o};
        }
        if (dc >= 0.f) out[m++] = cur;
        prev = cur;
        dp = dc;
    }
    return m;
}

// Rotated IoU of two BEV rectangles (cx, cy, w, h, angle_deg): the quantity detectron2's single_box_iou_rotated
// (box_iou_rotated_utils.h) defines -- corners centre +- (w/2) (cos, -sin) +- (h/2) (sin, cos), zero below 1e-14 m^2 of
// area -- computed by clipping b2 against b1 in b1's own frame, where b1 is the axis-aligned [-w1/2, w1/2] x [-h1/2, h1/2]
// and b2 is turned by the angle difference alone.  So boxes of one yaw stay exactly axis-aligned and rectangles that
// share an edge, are nested or are the same box written another way (angle + 180, w <-> h with angle + 90) come out
// within float32 rounding of their float64 IoU; detectron2's float32 edge-intersection test (|det| <= 1e-14 on metre
// scale edges) and its contracted hull test do not.  sincospif is exact at multiples of 90 degrees.
__device__ float rotated_iou(const float* b1, const float* b2) {
    const float a1 = b1[2] * b1[3], a2 = b2[2] * b2[3];
    if (a1 < 1e-14f || a2 < 1e-14f) return 0.f;
    float s1, c1, s, c;
    sincospif(b1[4] / 180.f, &s1, &c1);
    sincospif((b2[4] - b1[4]) / 180.f, &s, &c);
    const float dx = b2[0] - b1[0], dy = b2[1] - b1[1];
    const float X = dx * c1 - dy * s1, Y = dx * s1 + dy * c1;  // b2's centre on b1's width / length axes
    const float hw = 0.5f * b2[2], hh = 0.5f * b2[3];
    const float ux = c * hw, uy = -s * hw, vx = s * hh, vy = c * hh;
    P2 buf[2][kClipMax];
    buf[0][0] = {X + ux + vx, Y + uy + vy};
    buf[0][1] = {X + ux - vx, Y + uy - vy};
    buf[0][2] = {X - ux - vx, Y - uy - vy};
    buf[0][3] = {X - ux + vx, Y - uy + vy};
    const float lx = 0.5f * b1[2], ly = 0.5f * b1[3];
    int n = clip_half_plane(buf[0], 4, buf[1], 0, 1.f, lx);
    n = clip_half_plane(buf[1], n, buf[0], 0, -1.f, lx);
    n = clip_half_plane(buf[0], n, buf[1], 1, 1.f, ly);
    n = clip_half_plane(buf[1], n, buf[0], 1, -1.f, ly);
    if (n <= 2) return 0.f;
    const P2* q = buf[0];
    float area2 = 0.f;
    for (int i = 1; i + 1 < n; ++i)
        area2 += (q[i].x - q[0].x) * (q[i + 1].y - q[0].y) - (q[i].y - q[0].y) * (q[i + 1].x - q[0].x);
    const float inter = fminf(0.5f * fabsf(area2), fminf(a1, a2));
    return inter / (a1 + a2 - inter);
}

__device__ void quat_to_mat3(const float* q, float* R) {  // pytorch3d quaternion_to_matrix, real-first
    const float r = q[0], i = q[1], j = q[2], k = q[3];
    const float two_s = 2.0f / (r * r + i * i + j * j + k * k);
    R[0] = 1.f - two_s * (j * j + k * k); R[1] = two_s * (i * j - k * r); R[2] = two_s * (i * k + j * r);
    R[3] = two_s * (i * j + k * r); R[4] = 1.f - two_s * (i * i + k * k); R[5] = two_s * (j * k - i * r);
    R[6] = two_s * (i * k - j * r); R[7] = two_s * (j * k + i * r); R[8] = 1.f - two_s * (i * i + j * j);
}

// pytorch3d matrix_to_quaternion (rotation_conversions.py): best-conditioned of the four candidates, real part first,
// no sign standardisation -- the quaternion the reference stores in pred_boxes3d_global (postprocessing.py:43-46).
__device__ void mat3_to_quat(const float* m, float* q) {
    const float arg[4] = {1.f + m[0] + m[4] + m[8], 1.f + m[0] - m[4] - m[8], 1.f - m[0] + m[4] - m[8],
                          1.f - m[0] - m[4] + m[8]};
    float qa[4];
    int best = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        qa[i] = arg[i] > 0.f ? sqrtf(arg[i]) : 0.f;
        if (qa[i] > qa[best]) best = i;
    }
    const float c[4][4] = {{qa[0] * qa[0], m[7] - m[5], m[2] - m[6], m[3] - m[1]},
                           {m[7] - m[5], qa[1] * qa[1], m[3] + m[1], m[2] + m[6]},
                           {m[2] - m[6], m[3] + m[1], qa[2] * qa[2], m[5] + m[7]},
                           {m[3] - m[1], m[6] + m[2], m[7] + m[5], qa[3] * qa[3]}};
    const float den = 2.0f * fmaxf(qa[best], 0.1f);
#pragma unroll
    for (int i = 0; i < 4; ++i) q[i] = c[best][i] / den;
}

__device__ void invert_K(const float* K, float* iK) {  // adjugate in double, like decode.cu
    const double a = K[0], bb = K[1], c = K[2], d = K[3], e = K[4], f = K[5], g = K[6], h = K[7], i9 = K[8];
    const double A = e * i9 - f * h, Bc = -(d * i9 - f * g), Cc = d * h - e * g;
    const double rdet = 1.0 / (a * A + bb * Bc + c * Cc);
    iK[0] = static_cast<float>(A * rdet);
    iK[1] = static_cast<float>(-(bb * i9 - c * h) * rdet);
    iK[2] = static_cast<float>((bb * f - c * e) * rdet);
    iK[3] = static_cast<float>(Bc * rdet);
    iK[4] = static_cast<float>((a * i9 - c * g) * rdet);
    iK[5] = static_cast<float>(-(a * f - c * d) * rdet);
    iK[6] = static_cast<float>(Cc * rdet);
    iK[7] = static_cast<float>(-(a * h - bb * g) * rdet);
    iK[8] = static_cast<float>((a * e - bb * d) * rdet);
}

// One decoded box -> global rotation / translation (postprocessing.py:25-46) and its BEV top-surface rectangle
// (boxes3d.py:47-64, bev_nms.py:71-96).
__device__ void box_to_global(const Det& D, const float* iK, const float* Rw, const float* pose_t, float* R, float* t,
                              float* rect) {
    const float u = D.proj_ctr[0], v = D.proj_ctr[1];
    const float tv[3] = {(iK[0] * u + iK[1] * v + iK[2]) * D.depth, (iK[3] * u + iK[4] * v + iK[5]) * D.depth,
                         (iK[6] * u + iK[7] * v + iK[8]) * D.depth};
    float Rs[9];
    quat_to_mat3(D.quat, Rs);
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int cc = 0; cc < 3; ++cc) R[r * 3 + cc] = Rw[r * 3] * Rs[cc] + Rw[r * 3 + 1] * Rs[3 + cc] + Rw[r * 3 + 2] * Rs[6 + cc];
        t[r] = Rw[r * 3] * tv[0] + Rw[r * 3 + 1] * tv[1] + Rw[r * 3 + 2] * tv[2] + pose_t[r];
    }
    const float hl = 0.5f * D.size[1], hw = 0.5f * D.size[0], hh = 0.5f * D.size[2];  // (l, w, h) = size[1, 0, 2]
    // corners 0, 1, 5, 4 of the template: (+l,+w,+h), (+l,-w,+h), (-l,-w,+h), (-l,+w,+h)
    const float sx[4] = {hl, hl, -hl, -hl}, sy[4] = {hw, -hw, -hw, hw};
    float bx[4], by[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float X = R[0] * sx[k] + R[1] * sy[k] + R[2] * hh + t[0];
        const float Y = R[3] * sx[k] + R[4] * sy[k] + R[5] * hh + t[1];
        bx[k] = -Y;  // VEHICLE_TO_BEV_ROTATION: (x, y)_bev = (-Y, -X)
        by[k] = -X;
    }
    const float fx = bx[0] - bx[3], fy = by[0] - by[3];
    rect[0] = 0.5f * (bx[0] + bx[2]);
    rect[1] = 0.5f * (by[0] + by[2]);
    rect[2] = sqrtf((bx[0] - bx[1]) * (bx[0] - bx[1]) + (by[0] - by[1]) * (by[0] - by[1]));  // width
    rect[3] = sqrtf(fx * fx + fy * fy);                                                        // length
    rect[4] = atan2f(fx, fy) * 57.29577951308232f;
}

// Rectangles whose bounding circles are apart (with a relative margin far above fp32 rounding) are disjoint: their IoU is
// exactly 0 in the polygon clipper as well, so for iou_thresh >= 0 the pair never suppresses and needs no clipping.
__device__ __forceinline__ bool circles_apart(const float* a, const float* b) {
    const float ra = 0.5f * sqrtf(a[2] * a[2] + a[3] * a[3]), rb = 0.5f * sqrtf(b[2] * b[2] + b[3] * b[3]);
    const float dx = a[0] - b[0], dy = a[1] - b[1], r = (ra + rb) * 1.001f + 1e-4f;
    return dx * dx + dy * dy > r * r;
}

}  // namespace

}  // namespace dd3d
