// The per-detection inverse transform of a test-time-augmentation view, shared by the one-CTA merge (tta.cu) and the
// multi-CTA merge for large sets (tta_large.cu).  See tta.cu for the reference lines each step restates.
#pragma once
#include "detect.cuh"

namespace dd3d {

__device__ __forceinline__ void tta_inv3(const float* K, float* iK) {  // adjugate in double like decode.cu
    const double a = K[0], b = K[1], c = K[2], d = K[3], e = K[4], f = K[5], g = K[6], h = K[7], i = K[8];
    const double A = e * i - f * h, B = -(d * i - f * g), C = d * h - e * g;
    const double r = 1.0 / (a * A + b * B + c * C);
    iK[0] = static_cast<float>(A * r);
    iK[1] = static_cast<float>(-(b * i - c * h) * r);
    iK[2] = static_cast<float>((b * f - c * e) * r);
    iK[3] = static_cast<float>(B * r);
    iK[4] = static_cast<float>((a * i - c * g) * r);
    iK[5] = static_cast<float>(-(a * f - c * d) * r);
    iK[6] = static_cast<float>(C * r);
    iK[7] = static_cast<float>(-(a * h - b * g) * r);
    iK[8] = static_cast<float>((a * e - b * d) * r);
}

// Detection d of view `a` (iK = inverse of V.K_view) mapped back to the original image, in place.
__device__ __forceinline__ void tta_invert_det(Det& d, const TtaView& V, const float* iK, int a) {
    // ---- 2-D box: inverse transforms in reverse order, each in fp32 (fvcore apply_box = 4 corners -> min / max)
    float x1 = d.box[0], y1 = d.box[1], x2 = d.box[2], y2 = d.box[3];
    if (V.flip) {
        const float nx1 = V.view_w - x2, nx2 = V.view_w - x1;
        x1 = nx1;
        x2 = nx2;
    }
#pragma unroll
    for (int s = 0; s < 2; ++s) {  // un-resize view -> input, then input -> original
        x1 *= V.inv_sx[s];
        x2 *= V.inv_sx[s];
        y1 *= V.inv_sy[s];
        y2 *= V.inv_sy[s];
    }
    d.box[0] = fminf(x1, x2);
    d.box[1] = fminf(y1, y2);
    d.box[2] = fmaxf(x1, x2);
    d.box[3] = fmaxf(y1, y2);
    // ---- 3-D box: camera-frame translation of the view (Boxes3D.tvec), mirror if flipped
    const float u = d.proj_ctr[0], v = d.proj_ctr[1];
    float tx = (iK[0] * u + iK[1] * v + iK[2]) * d.depth;
    const float ty = (iK[3] * u + iK[4] * v + iK[5]) * d.depth;
    const float tz = (iK[6] * u + iK[7] * v + iK[8]) * d.depth;
    if (V.flip) {
        const float q0 = d.quat[0], q1 = d.quat[1], q2 = d.quat[2], q3 = d.quat[3];
        d.quat[0] = q3;
        d.quat[1] = -q2;
        d.quat[2] = -q1;
        d.quat[3] = q0;
        tx = -tx;
    }
    // ---- Boxes3D.from_vectors with the recovered original intrinsics: proj_ctr = (K t)[:2] / (K t)[2], depth = t.z
    const float* K = V.K_orig;
    const float px = K[0] * tx + K[1] * ty + K[2] * tz;
    const float py = K[3] * tx + K[4] * ty + K[5] * tz;
    const float pz = K[6] * tx + K[7] * ty + K[8] * tz;
    d.proj_ctr[0] = px / pz;
    d.proj_ctr[1] = py / pz;
    d.depth = tz;
    d.level = a;  // the view the detection came from (the merged Instances carry no fpn_levels)
}

}  // namespace dd3d
