// Dense threshold -> exact per-(image, level) top-k -> fused 2-D / 3-D box decode.
//
// Replaces FCOS2DInference.forward_for_single_feature_map (reference fcos2d.py:270-344) and
// FCOS3DInference.forward_for_single_feature_map + predictions_to_boxes3d + allocentric_to_egocentric
// (fcos3d.py:328-399, :16-52; geometry.py:15-55, 86-112), i.e. ~55 tiny ATen kernels and 2 host syncs per
// image x level in the reference, with 4 launches for the whole batch and no host sync.
//
//   1. score_hist   : s = sigmoid(logit) * sigmoid(ctr);  s > thresh  -> histogram of the float bits of s
//   2. select       : per (image, level) find the histogram bin T holding the k-th largest score
//   3. compact      : candidates in bins > T are certainly in the top-k ("sure"); bin == T goes to "boundary"
//   4. finalize     : exact rank inside the boundary bin (score desc, index asc) -- from the boundary buffer, or, when more
//                     than kBoundaryCap candidates share that bin, by re-reading the level (select_overflow) -- then one
//                     thread per survivor gathers its 4 + 11 regression values and decodes the 2-D box and the 3-D box.
// The result is exactly the first PRE_NMS_TOPK candidates in (score desc, index asc) order, for every input.
// Set semantics match `topk(sorted=False)` (fcos2d.py:312-313); order is fixed later by the NMS sort.
#include "detect.cuh"
#include "pdl.cuh"

#include <math.h>
#include <string.h>

namespace dd3d {

namespace {

constexpr int kDenseThreads = 256;
constexpr float kEps = 1e-7f;

__device__ __forceinline__ int find_level(const DecodeParams& p, int blk) {
    int l = 0;
#pragma unroll
    for (int i = 1; i < kLevels; ++i)
        if (i < p.num_levels && blk >= p.lvl[i].block_begin) l = i;
    return l;
}

// key of a score above the threshold: its float bits relative to the threshold's; bin = key >> hist_shift.  Every ranked
// score is <= 1.0f (a product of two sigmoids), so the bin stays below kHistBins (decode_finalize_params picks the shift).
__device__ __forceinline__ uint32_t score_key(const DecodeParams& p, float s) { return __float_as_uint(s) - p.thresh_bits; }

__device__ __forceinline__ int score_bin(const DecodeParams& p, float s) {
    return static_cast<int>(score_key(p, s) >> p.hist_shift);
}

// Calls f(class, s) for every class of pixel `pix` (< H * W) of image b at level L whose thresholded score passes, in class
// order; s = sigmoid(cls) * sigmoid(ctr) is the ranked score.  Pixels where no class passes alone are skipped before the
// centerness is read (class_passes): under the sparse box2d tower their box map rows hold stale workspace.
template <class F>
__device__ __forceinline__ void for_each_candidate(const DecodeParams& p, const DecodeLevel& L, int b, int pix, F&& f) {
    const size_t gp = static_cast<size_t>(b) * (L.H * L.W) + pix;
    const float* lg = L.cls + gp * p.cls_pitch;
    if (!class_passes(lg, p.C, p.thresh)) return;
    const float ctr = sigmoidf(__ldg(L.box + gp * 16 + 4));
    for (int c0 = 0; c0 < p.C; c0 += 4) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(lg + c0));
        const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int c = c0 + j;
            if (c < p.C) {
                const float cs = sigmoidf(vv[j]);
                const float s = cs * ctr;
                if ((p.thresh_with_ctr ? s : cs) > p.thresh) f(c, s);
            }
        }
    }
}

// mode 0: histogram, mode 1: compaction
template <int MODE>
__global__ void __launch_bounds__(kDenseThreads) dense_kernel(const __grid_constant__ DecodeParams p) {
    DD3D_PDL_PROLOGUE();
    __shared__ uint32_t shist[MODE == 0 ? kHistBins : 1];
    const int l = find_level(p, blockIdx.x);
    const DecodeLevel& L = p.lvl[l];
    const int b = blockIdx.y;
    const int hw = L.H * L.W;
    const int pix = (blockIdx.x - L.block_begin) * kDenseThreads + threadIdx.x;
    const int bl = b * p.num_levels + l;
    if (MODE == 0) {
        for (int i = threadIdx.x; i < kHistBins; i += kDenseThreads) shist[i] = 0;
        __syncthreads();
    }
    int T = 0;
    if (MODE == 1) T = p.sel[bl * 4 + 0];
    if (pix < hw) {
        for_each_candidate(p, L, b, pix, [&](int c, float s) {
            const int bin = min(score_bin(p, s), kHistBins - 1);
            if (MODE == 0) {
                atomicAdd(&shist[bin], 1u);
            } else {
                const uint2 rec = make_uint2(__float_as_uint(s), static_cast<uint32_t>(pix * p.C + c));
                if (bin > T) {
                    const int slot = atomicAdd(&p.counters[bl * 2 + 0], 1);
                    if (slot < p.topk) p.sure[static_cast<size_t>(bl) * p.topk + slot] = rec;
                } else if (bin == T) {
                    const int slot = atomicAdd(&p.counters[bl * 2 + 1], 1);
                    if (slot < kBoundaryCap) p.boundary[static_cast<size_t>(bl) * kBoundaryCap + slot] = rec;
                }
            }
        });
    }
    if (MODE == 0) {
        __syncthreads();
        uint32_t* gh = p.hist + static_cast<size_t>(bl) * kHistBins;
        for (int i = threadIdx.x; i < kHistBins; i += kDenseThreads) {
            const uint32_t v = shist[i];
            if (v) atomicAdd(&gh[i], v);
        }
    }
}

// One block per (level, image): locate the bin of the k-th largest score.
__global__ void __launch_bounds__(256) select_kernel(const __grid_constant__ DecodeParams p) {
    DD3D_PDL_PROLOGUE();
    __shared__ uint32_t chunk[256];
    const int bl = blockIdx.y * p.num_levels + blockIdx.x;
    const uint32_t* gh = p.hist + static_cast<size_t>(bl) * kHistBins;
    constexpr int per = kHistBins / 256;
    uint32_t loc = 0;
    for (int i = 0; i < per; ++i) loc += gh[threadIdx.x * per + i];
    chunk[threadIdx.x] = loc;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t total = 0;
        for (int i = 0; i < 256; ++i) total += chunk[i];
        int* sel = p.sel + bl * 4;
        sel[3] = static_cast<int>(total);
        if (total <= static_cast<uint32_t>(p.topk)) {
            sel[0] = -1;  // everything above the threshold survives
            sel[1] = static_cast<int>(total);
            sel[2] = 0;
        } else {
            uint32_t cum = 0;
            int ch = 255;
            for (; ch >= 0; --ch) {
                if (cum + chunk[ch] >= static_cast<uint32_t>(p.topk)) break;
                cum += chunk[ch];
            }
            int bin = ch * per + per - 1;
            for (;; --bin) {
                const uint32_t h = gh[bin];
                if (cum + h >= static_cast<uint32_t>(p.topk)) break;
                cum += h;
            }
            sel[0] = bin;
            sel[1] = static_cast<int>(cum);           // strictly above bin T
            sel[2] = p.topk - static_cast<int>(cum);  // still needed from bin T
        }
    }
}

struct Mat3 {
    float m[9];
};

__device__ __forceinline__ Mat3 invert_intrinsics(const float* K) {
    // adjugate / determinant in double, rounded once to fp32 (reference: torch.inverse, core.py:93)
    const double a = K[0], b = K[1], c = K[2], d = K[3], e = K[4], f = K[5], g = K[6], h = K[7], i = K[8];
    const double A = e * i - f * h, Bc = -(d * i - f * g), Cc = d * h - e * g;
    const double det = a * A + b * Bc + c * Cc;
    const double r = 1.0 / det;
    Mat3 o;
    o.m[0] = static_cast<float>(A * r);
    o.m[1] = static_cast<float>(-(b * i - c * h) * r);
    o.m[2] = static_cast<float>((b * f - c * e) * r);
    o.m[3] = static_cast<float>(Bc * r);
    o.m[4] = static_cast<float>((a * i - c * g) * r);
    o.m[5] = static_cast<float>(-(a * f - c * d) * r);
    o.m[6] = static_cast<float>(Cc * r);
    o.m[7] = static_cast<float>(-(a * h - b * g) * r);
    o.m[8] = static_cast<float>((a * e - b * d) * r);
    return o;
}

__device__ __forceinline__ void unproject(const Mat3& iK, float u, float v, float* ray) {
    ray[0] = iK.m[0] * u + iK.m[1] * v + iK.m[2];
    ray[1] = iK.m[3] * u + iK.m[4] * v + iK.m[5];
    ray[2] = iK.m[6] * u + iK.m[7] * v + iK.m[8];
}

// pytorch3d quaternion_to_matrix (real-first)
__device__ __forceinline__ void quat_to_mat(const float* q, float* R) {
    const float r = q[0], i = q[1], j = q[2], k = q[3];
    const float two_s = 2.0f / (r * r + i * i + j * j + k * k);
    R[0] = 1.f - two_s * (j * j + k * k);
    R[1] = two_s * (i * j - k * r);
    R[2] = two_s * (i * k + j * r);
    R[3] = two_s * (i * j + k * r);
    R[4] = 1.f - two_s * (i * i + k * k);
    R[5] = two_s * (j * k - i * r);
    R[6] = two_s * (i * k - j * r);
    R[7] = two_s * (j * k + i * r);
    R[8] = 1.f - two_s * (i * i + j * j);
}

// pytorch3d (>= 0.5) matrix_to_quaternion: best-conditioned candidate, no sign standardisation
__device__ __forceinline__ void mat_to_quat(const float* m, float* q) {
    const float m00 = m[0], m01 = m[1], m02 = m[2], m10 = m[3], m11 = m[4], m12 = m[5], m20 = m[6], m21 = m[7],
                m22 = m[8];
    float arg[4] = {1.f + m00 + m11 + m22, 1.f + m00 - m11 - m22, 1.f - m00 + m11 - m22, 1.f - m00 - m11 + m22};
    float qa[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) qa[t] = arg[t] > 0.f ? sqrtf(arg[t]) : 0.f;
    int best = 0;
#pragma unroll
    for (int t = 1; t < 4; ++t)
        if (qa[t] > qa[best]) best = t;  // first maximum, like argmax
    float c[4];
    if (best == 0) {
        c[0] = qa[0] * qa[0]; c[1] = m21 - m12; c[2] = m02 - m20; c[3] = m10 - m01;
    } else if (best == 1) {
        c[0] = m21 - m12; c[1] = qa[1] * qa[1]; c[2] = m10 + m01; c[3] = m02 + m20;
    } else if (best == 2) {
        c[0] = m02 - m20; c[1] = m10 + m01; c[2] = qa[2] * qa[2]; c[3] = m12 + m21;
    } else {
        c[0] = m10 - m01; c[1] = m20 + m02; c[2] = m21 + m12; c[3] = qa[3] * qa[3];
    }
    const float den = 2.0f * fmaxf(qa[best], 0.1f);
#pragma unroll
    for (int t = 0; t < 4; ++t) q[t] = c[t] / den;
}

// g3d: the candidate pixel's box3d predictor outputs (dense map pixel or sparse row), channel = component * C3 + class
__device__ void decode_one(const DecodeParams& p, const DecodeLevel& L, int b, int l, uint32_t score_bits, int index,
                           const float* g3d, Det* out) {
    const int hw = L.H * L.W;
    const int pix = index / p.C;
    const int c = index - pix * p.C;
    const int py = pix / L.W, px = pix - py * L.W;
    float lx = static_cast<float>(px * L.stride), ly = static_cast<float>(py * L.stride);
    if (p.loc_offset_half) {
        lx += static_cast<float>(L.stride / 2);
        ly += static_cast<float>(L.stride / 2);
    }
    const size_t gp = static_cast<size_t>(b) * hw + pix;
    const float4 reg = __ldg(reinterpret_cast<const float4*>(L.box + gp * 16));
    Det d;
    d.box[0] = lx - reg.x;
    d.box[1] = ly - reg.y;
    d.box[2] = lx + reg.z;
    d.box[3] = ly + reg.w;
    const float s = __uint_as_float(score_bits);
    d.score = sqrtf(s);
    d.cls = c;
    d.level = l;
    d.loc[0] = lx;
    d.loc[1] = ly;
    d.index = index;
    d.attr = 0;
    d.speed = 0.f;
    d.pad = 0;
    if (p.attr_off >= 0) {  // NuscenesInference (nuscenes_dd3d.py:268-298): first maximum like torch.argmax
        const float* a = L.cls + gp * p.cls_pitch + p.attr_off;
        float best = __ldg(a);
        for (int t = 1; t < p.num_attr; ++t) {
            const float v = __ldg(a + t);
            if (v > best) {
                best = v;
                d.attr = t;
            }
        }
        d.speed = __ldg(a + p.num_attr);
    }

    if (!p.box3d_on) {  // 2-D detector only (core.py:117-125): the NMS is keyed on `scores`
        d.score3d = d.score;
#pragma unroll
        for (int t = 0; t < 4; ++t) d.quat[t] = t == 0 ? 1.f : 0.f;
        d.proj_ctr[0] = lx;
        d.proj_ctr[1] = ly;
        d.depth = 0.f;
#pragma unroll
        for (int t = 0; t < 3; ++t) d.size[t] = 0.f;
        *out = d;
        return;
    }
    // channel = component * C3 + class (class 0 when class agnostic; fcos3d.py:333-352); the class-gathered rows hold the
    // candidate's own class only
    const int C = p.b3d_by_class ? 1 : p.C3;
    const float* g = g3d + (C == 1 ? 0 : c);
    float q[4] = {__ldg(g), __ldg(g + C), __ldg(g + 2 * C), __ldg(g + 3 * C)};
    const float cx = __ldg(g + 4 * C), cy = __ldg(g + 5 * C);
    float depth = __ldg(g + 6 * C);
    const float sz[3] = {__ldg(g + 7 * C), __ldg(g + 8 * C), __ldg(g + 9 * C)};
    const float conf = sigmoidf(__ldg(g + 10 * C));
    d.score3d = d.score * conf;

    // fcos3d.py:31-34
    float n = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    n = fmaxf(n, kEps);
#pragma unroll
    for (int t = 0; t < 4; ++t) q[t] = q[t] / n;
    n = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
#pragma unroll
    for (int t = 0; t < 4; ++t) q[t] = q[t] / n;

    const Mat3 iK = invert_intrinsics(p.K + b * 9);
    if (p.scale_depth_by_focal) {  // fcos3d.py:36-38
        const float pixel_size = sqrtf(iK.m[0] * iK.m[0] + iK.m[4] * iK.m[4]);
        depth = depth / (pixel_size * p.depth_factor);
    }
    if (p.predict_distance) {  // fcos3d.py:40-41
        float r[3];
        unproject(iK, lx, ly, r);
        depth = depth / fmaxf(sqrtf(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]), kEps);
    }
    depth = fminf(fmaxf(depth, p.min_depth), p.max_depth);
    const float pcx = cx + lx, pcy = cy + ly;

    if (p.allocentric) {  // geometry.py:15-55
        float Ro[9];
        quat_to_mat(q, Ro);
        float ray[3];
        unproject(iK, pcx, pcy, ray);
        const float rn = sqrtf(ray[0] * ray[0] + ray[1] * ray[1] + ray[2] * ray[2]);
        const float z[3] = {ray[0] / rn, ray[1] / rn, ray[2] / rn};
        float y[3] = {0.f - z[1] * z[0], 1.f - z[1] * z[1], 0.f - z[1] * z[2]};
        const float yn = sqrtf(y[0] * y[0] + y[1] * y[1] + y[2] * y[2]);
        y[0] /= yn; y[1] /= yn; y[2] /= yn;
        const float x[3] = {y[1] * z[2] - y[2] * z[1], y[2] * z[0] - y[0] * z[2], y[0] * z[1] - y[1] * z[0]};
        // R_local_to_global = [x y z] as columns;  R = R_l2g @ R_obj
        float R[9];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
#pragma unroll
            for (int cc = 0; cc < 3; ++cc)
                R[r * 3 + cc] = x[r] * Ro[0 * 3 + cc] + y[r] * Ro[1 * 3 + cc] + z[r] * Ro[2 * 3 + cc];
        }
        mat_to_quat(R, q);
        const float qn = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
        if (fabsf(qn - 1.0f) > 1e-3f + 1e-5f) {
            const float dn = fmaxf(qn, kEps);
#pragma unroll
            for (int t = 0; t < 4; ++t) q[t] = q[t] / dn;
        }
    }
#pragma unroll
    for (int t = 0; t < 4; ++t) d.quat[t] = q[t];
    d.proj_ctr[0] = pcx;
    d.proj_ctr[1] = pcy;
    d.depth = depth;
#pragma unroll
    for (int t = 0; t < 3; ++t) d.size[t] = (tanhf(sz[t]) + 1.0f) * __ldg(p.canon + c * 3 + t);  // fcos3d.py:50
    *out = d;
}

constexpr int kSelectThreads = 256;

// Exclusive prefix sum over the CTA (kSelectThreads threads, all of them call it); *total = the sum of all v.
__device__ uint32_t block_exclusive_scan(uint32_t v, uint32_t* s_warp /* [kSelectThreads / 32 + 1] */, uint32_t* total) {
    constexpr int kWarps = kSelectThreads / 32;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t acc = 0;
        for (int w = 0; w < kWarps; ++w) {
            const uint32_t t = s_warp[w];
            s_warp[w] = acc;
            acc += t;
        }
        s_warp[kWarps] = acc;
    }
    __syncthreads();
    const uint32_t r = s_warp[warp] + incl - v;
    *total = s_warp[kWarps];
    __syncthreads();  // s_warp is reused by the next call
    return r;
}

// Bin T of (image b, level l) holds more candidates than the boundary buffer (scores clustered in one bin, or tied): the CTA
// ranks it by re-reading the level instead.  Histogram passes over the next bits of the key (11 per pass: two passes for the
// widest bins, 2^19 ulps) narrow bin T down to the one score value V of the k-th candidate; a last pass takes every
// candidate of bin T above V (out[0, n_above), pixel order) and the first `need_v` ties at V in index order
// (out[n_above, need), by a CTA scan per 256-pixel chunk, which visits the (pixel, class) pairs in index order).
// Same set as the boundary ranking (score desc, index asc); off the common path, which never has more than kBoundaryCap.
__device__ void select_overflow(const DecodeParams& p, int b, int l, uint32_t T, int need, uint2* out) {
    __shared__ uint32_t h[kHistBins];
    __shared__ uint32_t s_warp[kSelectThreads / 32 + 1];
    __shared__ uint32_t s_prefix;
    __shared__ int s_need;
    const DecodeLevel& L = p.lvl[l];
    const int hw = L.H * L.W;
    const int need_total = need;
    uint32_t prefix = T;  // key >> shift of the candidates still in play
    for (int shift = p.hist_shift; shift > 0;) {
        const int bits = min(shift, 11), nshift = shift - bits;
        const uint32_t nbins = 1u << bits;
        for (uint32_t i = threadIdx.x; i < nbins; i += blockDim.x) h[i] = 0;
        __syncthreads();
        for (int pix = threadIdx.x; pix < hw; pix += blockDim.x) {
            for_each_candidate(p, L, b, pix, [&](int, float s) {
                const uint32_t key = score_key(p, s);
                if ((key >> shift) == prefix) atomicAdd(&h[(key >> nshift) & (nbins - 1)], 1u);
            });
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t cum = 0;
            int bin = static_cast<int>(nbins) - 1;
            for (; bin > 0; --bin) {
                if (cum + h[bin] >= static_cast<uint32_t>(need)) break;
                cum += h[bin];
            }
            s_prefix = (prefix << bits) | static_cast<uint32_t>(bin);
            s_need = need - static_cast<int>(cum);
        }
        __syncthreads();
        prefix = s_prefix;
        need = s_need;
        shift = nshift;
    }
    const uint32_t vkey = prefix;  // the k-th candidate's key; `need` ties at it are still taken
    const int n_above = need_total - need;
    uint32_t base_above = 0, base_tie = 0;
    for (int p0 = 0; p0 < hw; p0 += blockDim.x) {
        const int pix = p0 + threadIdx.x;
        uint32_t cnt = 0;  // (candidates above V << 16) | ties at V, of this pixel: <= C <= 128 each, < 2^16 per chunk
        if (pix < hw) {
            for_each_candidate(p, L, b, pix, [&](int, float s) {
                const uint32_t key = score_key(p, s);
                if ((key >> p.hist_shift) == T) cnt += key > vkey ? (1u << 16) : key == vkey ? 1u : 0u;
            });
        }
        uint32_t total;
        const uint32_t excl = block_exclusive_scan(cnt, s_warp, &total);
        if (cnt) {
            uint32_t a = base_above + (excl >> 16), t = base_tie + (excl & 0xffffu);
            for_each_candidate(p, L, b, pix, [&](int c, float s) {
                const uint32_t key = score_key(p, s);
                if ((key >> p.hist_shift) != T) return;
                const uint2 rec = make_uint2(__float_as_uint(s), static_cast<uint32_t>(pix * p.C + c));
                if (key > vkey) {
                    out[a++] = rec;
                } else if (key == vkey) {
                    if (t < static_cast<uint32_t>(need)) out[n_above + t] = rec;
                    ++t;
                }
            });
        }
        base_above += total >> 16;
        base_tie += total & 0xffffu;
    }
}

// One block per (level, image): the final candidate list.  Candidates in histogram bins above the k-th score's bin are in
// ("sure"); inside that bin the exact rank (score desc, index asc) decides.  fin[slot] = (score bits, index).
__global__ void __launch_bounds__(kSelectThreads) select_final_kernel(const __grid_constant__ DecodeParams p) {
    DD3D_PDL_PROLOGUE();
    const int l = blockIdx.x, b = blockIdx.y;
    const int bl = b * p.num_levels + l;
    const int* sel = p.sel + bl * 4;
    const int n_sure = min(p.counters[bl * 2 + 0], p.topk);
    const int nb_raw = p.counters[bl * 2 + 1];
    const int nb = min(nb_raw, kBoundaryCap);
    const bool overflow = sel[0] >= 0 && nb_raw > kBoundaryCap;
    const int need = sel[0] < 0 ? 0 : overflow ? sel[2] : min(sel[2], nb);
    if (threadIdx.x == 0) p.cand_count[bl] = n_sure + need;
    const uint2* sure = p.sure + static_cast<size_t>(bl) * p.topk;
    const uint2* bnd = p.boundary + static_cast<size_t>(bl) * kBoundaryCap;
    uint2* fin = p.fin + static_cast<size_t>(bl) * p.topk;
    for (int i = threadIdx.x; i < n_sure; i += blockDim.x) fin[i] = sure[i];
    if (overflow) {
        select_overflow(p, b, l, static_cast<uint32_t>(sel[0]), need, fin + n_sure);
    } else if (need > 0) {
        for (int i = threadIdx.x; i < nb; i += blockDim.x) {
            const uint2 me = bnd[i];
            int rank = 0;
            for (int j = 0; j < nb; ++j) {
                const uint2 o = bnd[j];
                rank += (o.x > me.x) || (o.x == me.x && o.y < me.y);
            }
            if (rank < need) fin[n_sure + rank] = me;
        }
    }
}

// One thread per final candidate: 2-D box + 3-D box decode.  kFinalSplit CTAs share a (level, image): the finest level
// holds most of the candidates, and one 256-thread CTA walking 600 - 1000 of them was 18 - 31 us of pure latency.
constexpr int kFinalSplit = 8, kFinalThreads = 128;
__global__ void __launch_bounds__(kFinalThreads) decode_final_kernel(const __grid_constant__ DecodeParams p) {
    DD3D_PDL_PROLOGUE();
    const int l = blockIdx.x / kFinalSplit, part = blockIdx.x % kFinalSplit, b = blockIdx.y;
    const int bl = b * p.num_levels + l;
    const int n = p.cand_count[bl];
    const DecodeLevel& L = p.lvl[l];
    const uint2* fin = p.fin + static_cast<size_t>(bl) * p.topk;
    Det* out = p.cand + static_cast<size_t>(bl) * p.topk;
    const size_t hw = static_cast<size_t>(L.H) * L.W;
    for (int i = part * kFinalThreads + threadIdx.x; i < n; i += kFinalSplit * kFinalThreads) {
        const uint2 me = fin[i];
        const float* g3d = nullptr;
        if (p.box3d_on) {
            // b3d_pitch is the row pitch of either sparse predictor (kB3dGatherPitch for the class-gathered one)
            g3d = p.b3d_rows != nullptr ? p.b3d_rows + (static_cast<size_t>(bl) * p.topk + i) * p.b3d_pitch
                                        : L.b3d + (static_cast<size_t>(b) * hw + me.y / p.C) * p.b3d_pitch;
        }
        decode_one(p, L, b, l, me.x, static_cast<int>(me.y), g3d, out + i);
    }
}

__global__ void clear_kernel(uint32_t* ptr, size_t nwords) {
    DD3D_PDL_PROLOGUE();
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < nwords;
         i += static_cast<size_t>(gridDim.x) * blockDim.x)
        ptr[i] = 0;
}

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

}  // namespace

// scratch layout: [hist | counters | flags(1 word + pad)] (cleared every forward) then sel, sure, boundary, cand, cand_count
size_t decode_scratch_bytes(int B, int topk, int num_levels) {
    const size_t bl = static_cast<size_t>(B) * num_levels;
    size_t n = 0;
    n += align_up(bl * kHistBins * 4, 256);
    n += align_up(bl * 2 * 4, 256);
    n += 256;
    n += align_up(bl * 4 * 4, 256);
    n += align_up(bl * topk * 8, 256);
    n += align_up(bl * kBoundaryCap * 8, 256);
    n += align_up(bl * topk * sizeof(Det), 256);
    n += align_up(bl * 4, 256);
    n += align_up(bl * topk * 8, 256);  // fin
    return n;
}

void decode_bind_scratch(DecodeParams* p, void* scratch) {
    const size_t bl = static_cast<size_t>(p->B) * p->num_levels;
    uint8_t* s = static_cast<uint8_t*>(scratch);
    p->hist = reinterpret_cast<uint32_t*>(s);
    s += align_up(bl * kHistBins * 4, 256);
    p->counters = reinterpret_cast<int32_t*>(s);
    s += align_up(bl * 2 * 4, 256);
    p->flags = reinterpret_cast<int32_t*>(s);
    s += 256;
    p->sel = reinterpret_cast<int32_t*>(s);
    s += align_up(bl * 4 * 4, 256);
    p->sure = reinterpret_cast<uint2*>(s);
    s += align_up(bl * p->topk * 8, 256);
    p->boundary = reinterpret_cast<uint2*>(s);
    s += align_up(bl * kBoundaryCap * 8, 256);
    p->cand = reinterpret_cast<Det*>(s);
    s += align_up(bl * p->topk * sizeof(Det), 256);
    p->cand_count = reinterpret_cast<int32_t*>(s);
    s += align_up(bl * 4, 256);
    p->fin = reinterpret_cast<uint2*>(s);
}

void decode_finalize_params(DecodeParams* p) {
    int blk = 0;
    for (int l = 0; l < p->num_levels; ++l) {
        p->lvl[l].block_begin = blk;
        blk += (p->lvl[l].H * p->lvl[l].W + kDenseThreads - 1) / kDenseThreads;
    }
    p->total_blocks = blk;
    uint32_t tb;
    // the ranked score cls * ctr is > thresh only when the threshold is applied to the product; otherwise it can be anywhere
    // in (0, 1) and the histogram starts at 0
    float t = (p->thresh > 0.f && p->thresh_with_ctr) ? p->thresh : 0.f;
    memcpy(&tb, &t, 4);
    p->thresh_bits = tb;
    const uint32_t one = 0x3F800000u;
    int shift = 0;
    while (((one - tb) >> shift) >= static_cast<uint32_t>(kHistBins)) ++shift;
    p->hist_shift = shift;
}

cudaError_t launch_decode_select(const DecodeParams& p, cudaStream_t stream) {
    if (p.num_levels < 1 || p.num_levels > kLevels) return cudaErrorInvalidValue;
    const size_t bl = static_cast<size_t>(p.B) * p.num_levels;
    const size_t clear_words = (align_up(bl * kHistBins * 4, 256) + align_up(bl * 2 * 4, 256) + 256) / 4;
    cudaError_t e = launch_pdl(clear_kernel, dim3(148), dim3(256), 0, stream, p.hist, clear_words);
    dim3 dgrid(p.total_blocks, p.B);
    if (e == cudaSuccess) e = launch_pdl(dense_kernel<0>, dgrid, dim3(kDenseThreads), 0, stream, p);
    if (e == cudaSuccess) e = launch_pdl(select_kernel, dim3(p.num_levels, p.B), dim3(256), 0, stream, p);
    if (e == cudaSuccess) e = launch_pdl(dense_kernel<1>, dgrid, dim3(kDenseThreads), 0, stream, p);
    if (e == cudaSuccess) e = launch_pdl(select_final_kernel, dim3(p.num_levels, p.B), dim3(kSelectThreads), 0, stream, p);
    return e;
}

cudaError_t launch_decode_final(const DecodeParams& p, cudaStream_t stream) {
    if (p.num_levels < 1 || p.num_levels > kLevels) return cudaErrorInvalidValue;
    return launch_pdl(decode_final_kernel, dim3(p.num_levels * kFinalSplit, p.B), dim3(kFinalThreads), 0, stream, p);
}

cudaError_t launch_decode(const DecodeParams& p, cudaStream_t stream) {
    cudaError_t e = launch_decode_select(p, stream);
    if (e != cudaSuccess) return e;
    return launch_decode_final(p, stream);
}

}  // namespace dd3d
