// Rotated-box geometry shared by the BEV NMS kernels (bev_nms.cu, bev_nms_group.cu): detectron2's rotated IoU
// (box_iou_rotated_utils.h), pytorch3d's quaternion <-> matrix conversions and the decoded box -> global frame -> BEV
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
__device__ __forceinline__ float cross2(P2 a, P2 b) { return a.x * b.y - a.y * b.x; }
__device__ __forceinline__ float dot2(P2 a, P2 b) { return a.x * b.x + a.y * b.y; }
__device__ __forceinline__ P2 sub2(P2 a, P2 b) { return {a.x - b.x, a.y - b.y}; }

// detectron2 box_iou_rotated_utils.h: get_rotated_vertices
__device__ void rect_vertices(float x, float y, float w, float h, float a, P2* p) {
    const float th = a * 0.01745329251994329577f;
    const float c = cosf(th) * 0.5f, s = sinf(th) * 0.5f;
    p[0] = {x + s * h + c * w, y + c * h - s * w};
    p[1] = {x - s * h + c * w, y - c * h - s * w};
    p[2] = {2.f * x - p[0].x, 2.f * y - p[0].y};
    p[3] = {2.f * x - p[1].x, 2.f * y - p[1].y};
}

// get_intersection_points: edge x edge intersections + vertices of one rectangle inside the other (<= 24 points)
__device__ int intersection_points(const P2* p1, const P2* p2, P2* out) {
    P2 v1[4], v2[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        v1[i] = sub2(p1[(i + 1) & 3], p1[i]);
        v2[i] = sub2(p2[(i + 1) & 3], p2[i]);
    }
    int n = 0;
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            const float det = cross2(v2[j], v1[i]);
            if (fabsf(det) <= 1e-14f) continue;
            const P2 v12 = sub2(p2[j], p1[i]);
            const float t1 = cross2(v2[j], v12) / det, t2 = cross2(v1[i], v12) / det;
            if (t1 >= 0.f && t1 <= 1.f && t2 >= 0.f && t2 <= 1.f) out[n++] = {p1[i].x + v1[i].x * t1, p1[i].y + v1[i].y * t1};
        }
    {
        const P2 AB = v2[0], DA = v2[3];
        const float ABdotAB = dot2(AB, AB), ADdotAD = dot2(DA, DA);
        for (int i = 0; i < 4; ++i) {
            const P2 AP = sub2(p1[i], p2[0]);
            const float APdotAB = dot2(AP, AB), APdotAD = -dot2(AP, DA);
            if (APdotAB >= 0.f && APdotAD >= 0.f && APdotAB <= ABdotAB && APdotAD <= ADdotAD) out[n++] = p1[i];
        }
    }
    {
        const P2 AB = v1[0], DA = v1[3];
        const float ABdotAB = dot2(AB, AB), ADdotAD = dot2(DA, DA);
        for (int i = 0; i < 4; ++i) {
            const P2 AP = sub2(p2[i], p1[0]);
            const float APdotAB = dot2(AP, AB), APdotAD = -dot2(AP, DA);
            if (APdotAB >= 0.f && APdotAD >= 0.f && APdotAB <= ABdotAB && APdotAD <= ADdotAD) out[n++] = p2[i];
        }
    }
    return n;
}

// convex_hull_graham (shift_to_zero = true) followed by polygon_area
__device__ float hull_area(P2* q, int n) {
    int t = 0;
    for (int i = 1; i < n; ++i)
        if (q[i].y < q[t].y || (q[i].y == q[t].y && q[i].x < q[t].x)) t = i;
    const P2 start = q[t];
    for (int i = 0; i < n; ++i) q[i] = sub2(q[i], start);
    {
        const P2 tmp = q[0];
        q[0] = q[t];
        q[t] = tmp;
    }
    float dist[24];
    for (int i = 0; i < n; ++i) dist[i] = dot2(q[i], q[i]);
    // insertion sort of q[1..n) by polar angle around q[0] (ties: nearer first), as detectron2's CUDA path
    for (int i = 2; i < n; ++i) {
        const P2 qi = q[i];
        const float di = dist[i];
        int j = i - 1;
        while (j >= 1) {
            const float tmp = cross2(qi, q[j]);  // qi before q[j] ?
            const bool before = (fabsf(tmp) < 1e-6f) ? (di < dist[j]) : (tmp > 0.f);
            if (!before) break;
            q[j + 1] = q[j];
            dist[j + 1] = dist[j];
            --j;
        }
        q[j + 1] = qi;
        dist[j + 1] = di;
    }
    int k = 1;
    while (k < n && dist[k] <= 1e-8f) ++k;
    if (k == n) return 0.f;
    P2 hull[24];
    hull[0] = q[0];
    hull[1] = q[k];
    int m = 2;
    for (int i = k + 1; i < n; ++i) {
        while (m > 1 && cross2(sub2(q[i], hull[m - 2]), sub2(hull[m - 1], hull[m - 2])) >= 0.f) --m;
        hull[m++] = q[i];
    }
    if (m <= 2) return 0.f;
    float area = 0.f;
    for (int i = 1; i < m - 1; ++i) area += fabsf(cross2(sub2(hull[i], hull[0]), sub2(hull[i + 1], hull[0])));
    return area * 0.5f;
}

// single_box_iou_rotated; boxes are (cx, cy, w, h, angle_deg)
__device__ float rotated_iou(const float* b1, const float* b2) {
    const float a1 = b1[2] * b1[3], a2 = b2[2] * b2[3];
    if (a1 < 1e-14f || a2 < 1e-14f) return 0.f;
    const float sx = (b1[0] + b2[0]) * 0.5f, sy = (b1[1] + b2[1]) * 0.5f;  // shift centres for precision
    P2 p1[4], p2[4], pts[24];
    rect_vertices(b1[0] - sx, b1[1] - sy, b1[2], b1[3], b1[4], p1);
    rect_vertices(b2[0] - sx, b2[1] - sy, b2[2], b2[3], b2[4], p2);
    const int n = intersection_points(p1, p2, pts);
    if (n <= 2) return 0.f;
    const float inter = hull_area(pts, n);
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

}  // namespace

}  // namespace dd3d
