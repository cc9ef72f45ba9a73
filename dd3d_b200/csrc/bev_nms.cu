// Bird's-eye-view rotated NMS, one CTA per image (SURVEY.md 8f row 1).
//
// Replaces the reference's `DO_BEV_NMS` branch of DD3D.forward (core.py:137-151): nuscenes_sample_aggregate with one
// dummy group per image (postprocessing.py:58-108) -> sample_bev_nms (:22-55: boxes to the global frame through the
// image's pose) -> bev_nms (tridet/layers/bev_nms.py:99-133: top-surface rectangle in BEV, :51-96) -> detectron2
// batched_nms_rotated (polygon-clipping rotated IoU, greedy, class aware, score = scores_3d).
// Runs after the 2-D NMS / top-k kernel on its <= out_cap survivors (already sorted by scores_3d) and, like the
// reference, BEFORE detector_postprocess -- which this kernel then applies itself (scale, clip, drop empty).
#include "bev_geom.cuh"
#include "device_once.cuh"

namespace dd3d {

namespace {

constexpr int kBevMax = kBevNmsMax;
constexpr int kBevThreads = 128;

// ------------------------------------------------------------------------------------------------------------------
// NuscenesDD3D sample aggregation (nuscenes_dd3d.py:449-463 -> postprocessing.py:58-108): rotated NMS jointly over the
// cameras of one sample.  Kernel 1: one CTA per sample group (sort by scores_3d, pairwise IoU bit matrix, greedy scan);
// kernel 2: one CTA per image (cap on the survivors of the whole call, order-preserving compaction).
constexpr int kGrpMax = 768;      // boxes per sample group (6 cameras x out_cap 128)
constexpr int kGrpSort = 1024;
constexpr int kGrpThreads = 256;
constexpr int kGrpImages = 16;    // cameras per sample the kernel can hold
constexpr int kGrpWords = kGrpMax / 64;

struct AggParams {
    Det* dets;             // [B][cap]
    int32_t* counts;       // [B]
    const float* K;        // [B][9]
    const float* poses;    // [B][7]
    const int32_t* group;  // [B] sample group of each image
    float* global;         // [B][cap][10] : global quat (w,x,y,z), global tvec, size (pred_boxes3d_global)
    float* keep_score;     // [B][cap] scratch: scores_3d of the NMS survivors, -1 elsewhere
    int32_t* flags;        // bit 3: a group had more than kGrpMax boxes / kGrpImages images
    int B, cap, max_dets;
    float thr;
};

struct GrpSmem {
    unsigned long long mask[kGrpMax][kGrpWords];
    unsigned long long key[kGrpSort];
    float rect[kGrpMax][5];
    int cls[kGrpMax];
    uint32_t src[kGrpMax];  // image << 16 | slot
    int imgs[kGrpImages];
    int offs[kGrpImages + 1];
    int nimg;
};

__global__ void __launch_bounds__(kGrpThreads) sample_nms_kernel(const AggParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    GrpSmem& S = *reinterpret_cast<GrpSmem*>(smem_raw);
    const int g = blockIdx.x;
    if (threadIdx.x == 0) {
        int m = 0, total = 0;
        S.offs[0] = 0;
        for (int b = 0; b < p.B; ++b) {
            if (p.group[b] != g) continue;
            if (m == kGrpImages) {
                atomicOr(p.flags, 8);
                break;
            }
            int c = min(p.counts[b], p.cap);
            if (total + c > kGrpMax) {
                atomicOr(p.flags, 8);
                c = kGrpMax - total;
            }
            S.imgs[m] = b;
            total += c;
            S.offs[++m] = total;
        }
        S.nimg = m;
    }
    __syncthreads();
    const int nimg = S.nimg, n = S.offs[nimg];
    // ---- 1. boxes to the global frame, BEV rectangles, sort keys; keep_score = -1 on every slot of the group's images
    for (int m = 0; m < nimg; ++m)
        for (int s = threadIdx.x; s < p.cap; s += blockDim.x) p.keep_score[static_cast<size_t>(S.imgs[m]) * p.cap + s] = -1.0f;
    for (int i = threadIdx.x; i < kGrpSort; i += blockDim.x) S.key[i] = ~0ull;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        int m = 0;
        while (i >= S.offs[m + 1]) ++m;
        const int b = S.imgs[m], slot = i - S.offs[m];
        const Det& D = p.dets[static_cast<size_t>(b) * p.cap + slot];
        float iK[9], Rw[9], R[9], t[3], q[4];
        invert_K(p.K + b * 9, iK);
        quat_to_mat3(p.poses + b * 7, Rw);
        box_to_global(D, iK, Rw, p.poses + b * 7 + 4, R, t, S.rect[i]);
        mat3_to_quat(R, q);
        float* go = p.global + (static_cast<size_t>(b) * p.cap + slot) * 10;
        go[0] = q[0]; go[1] = q[1]; go[2] = q[2]; go[3] = q[3];
        go[4] = t[0]; go[5] = t[1]; go[6] = t[2];
        go[7] = D.size[0]; go[8] = D.size[1]; go[9] = D.size[2];
        S.cls[i] = D.cls;
        S.src[i] = (static_cast<uint32_t>(b) << 16) | static_cast<uint32_t>(slot);
        // descending scores_3d (non-negative floats order like their bit patterns), ties by concatenation index
        S.key[i] = (static_cast<unsigned long long>(~__float_as_uint(D.score3d)) << 32) | static_cast<unsigned>(i);
    }
    for (int i = threadIdx.x; i < kGrpMax * kGrpWords; i += blockDim.x) (&S.mask[0][0])[i] = 0ull;
    __syncthreads();
    // ---- 2. bitonic sort of the keys
    for (int k = 2; k <= kGrpSort; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < kGrpSort; i += blockDim.x) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const unsigned long long a = S.key[i], b2 = S.key[ixj];
                    const bool up = (i & k) == 0;
                    if ((a > b2) == up) {
                        S.key[i] = b2;
                        S.key[ixj] = a;
                    }
                }
            }
            __syncthreads();
        }
    // ---- 3. pairwise rotated IoU in sorted order (same class; same sample by construction)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int ri = warp; ri < n; ri += kGrpThreads / 32) {
        const int i = static_cast<int>(S.key[ri] & 0xffffffffull);
        for (int rj = ri + 1 + lane; rj < n; rj += 32) {
            const int j = static_cast<int>(S.key[rj] & 0xffffffffull);
            if (S.cls[i] == S.cls[j] && rotated_iou(S.rect[i], S.rect[j]) > p.thr)
                atomicOr(&S.mask[ri][rj >> 6], 1ull << (rj & 63));
        }
    }
    __syncthreads();
    // ---- 4. greedy scan; survivors publish their score
    if (threadIdx.x == 0) {
        unsigned long long removed[kGrpWords];
#pragma unroll
        for (int w = 0; w < kGrpWords; ++w) removed[w] = 0ull;
        for (int r = 0; r < n; ++r) {
            if ((removed[r >> 6] >> (r & 63)) & 1ull) continue;
#pragma unroll
            for (int w = 0; w < kGrpWords; ++w) removed[w] |= S.mask[r][w];
            const int i = static_cast<int>(S.key[r] & 0xffffffffull);
            const uint32_t src = S.src[i];
            const size_t at = static_cast<size_t>(src >> 16) * p.cap + (src & 0xffffu);
            p.keep_score[at] = p.dets[at].score3d;
        }
    }
}

__global__ void __launch_bounds__(kBevThreads) sample_compact_kernel(const AggParams p) {
    __shared__ unsigned char keep[kBevMax];
    __shared__ int new_pos[kBevMax];
    __shared__ int s_total;
    const int b = blockIdx.x;
    const int n = min(min(p.counts[b], p.cap), kBevMax);
    const size_t all = static_cast<size_t>(p.B) * p.cap;
    if (threadIdx.x == 0) s_total = 0;
    __syncthreads();
    // survivors of the whole call (keep = keep[:max_dets] is applied to the concatenation of ALL images of the call,
    // postprocessing.py:87-93)
    int part = 0;
    for (size_t i = threadIdx.x; i < all; i += blockDim.x) part += p.keep_score[i] >= 0.f;
    atomicAdd(&s_total, part);
    __syncthreads();
    const bool capped = p.max_dets > 0 && s_total > p.max_dets;
    __syncthreads();
    for (int s = threadIdx.x; s < kBevMax; s += blockDim.x) {
        bool k = false;
        if (s < n) {
            const size_t me = static_cast<size_t>(b) * p.cap + s;
            const float sc = p.keep_score[me];
            k = sc >= 0.f;
            if (k && capped) {  // rank among the survivors in the NMS output order: score desc, concatenation index asc
                int rank = 0;
                for (size_t i = 0; i < all; ++i) {
                    const float o = p.keep_score[i];
                    rank += (o > sc) || (o == sc && i < me);
                }
                k = rank < p.max_dets;
            }
        }
        keep[s] = k ? 1 : 0;
    }
    __syncthreads();
    Det mine[kBevMax / kBevThreads];
    float gl[kBevMax / kBevThreads][10];
    for (int s = 0; s < kBevMax / kBevThreads; ++s) {
        const int i = threadIdx.x + s * kBevThreads;
        if (i < n && keep[i]) {
            mine[s] = p.dets[static_cast<size_t>(b) * p.cap + i];
            const float* go = p.global + (static_cast<size_t>(b) * p.cap + i) * 10;
#pragma unroll
            for (int t = 0; t < 10; ++t) gl[s][t] = go[t];
        }
    }
    if (threadIdx.x == 0) {
        int m = 0;
        for (int i = 0; i < n; ++i) {
            new_pos[i] = m;
            m += keep[i];
        }
        s_total = m;
    }
    __syncthreads();
    for (int s = 0; s < kBevMax / kBevThreads; ++s) {
        const int i = threadIdx.x + s * kBevThreads;
        if (i < n && keep[i]) {
            p.dets[static_cast<size_t>(b) * p.cap + new_pos[i]] = mine[s];
            float* go = p.global + (static_cast<size_t>(b) * p.cap + new_pos[i]) * 10;
#pragma unroll
            for (int t = 0; t < 10; ++t) go[t] = gl[s][t];
        }
    }
    if (threadIdx.x == 0) p.counts[b] = s_total;
}

struct BevParams {
    Det* dets;             // [B][cap], compacted in place
    int32_t* counts;       // [B]
    const float* K;        // [B][9]
    const float* poses;    // [B][7] : pose quaternion (w, x, y, z) and translation (sensor -> global)
    const int32_t* sizes;  // [B][4] : h, w, out_h, out_w
    int32_t* flags;        // bit 2: more than kBevMax boxes
    int cap, do_postprocess;
    float thr;
};

__global__ void __launch_bounds__(kBevThreads) bev_nms_kernel(const BevParams p) {
    __shared__ float rect[kBevMax][5];
    __shared__ int cls[kBevMax];
    __shared__ unsigned long long mask[kBevMax][kBevMax / 64];
    __shared__ unsigned char keep[kBevMax];
    __shared__ int new_pos[kBevMax];
    __shared__ int s_total;
    const int b = blockIdx.x;
    int n = p.counts[b];
    if (n > kBevMax) {
        if (threadIdx.x == 0) atomicOr(p.flags, 4);
        n = kBevMax;
    }
    Det* dets = p.dets + static_cast<size_t>(b) * p.cap;
    // ---- 1. global-frame top-surface rectangles (postprocessing.py:25-46, boxes3d.py:47-64, bev_nms.py:71-96)
    const float* K = p.K + b * 9;
    const float* pose = p.poses + b * 7;
    float Rw[9];
    quat_to_mat3(pose, Rw);
    float iK[9];
    invert_K(K, iK);
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        float R[9], t[3];
        box_to_global(dets[i], iK, Rw, pose + 4, R, t, rect[i]);
        cls[i] = dets[i].cls;
    }
    for (int i = threadIdx.x; i < kBevMax * (kBevMax / 64); i += blockDim.x) (&mask[0][0])[i] = 0ull;
    __syncthreads();
    // ---- 2. pairwise rotated IoU (same class, j > i)
    for (int pidx = threadIdx.x; pidx < n * n; pidx += blockDim.x) {
        const int i = pidx / n, j = pidx - i * n;
        if (j > i && cls[i] == cls[j] && rotated_iou(rect[i], rect[j]) > p.thr)
            atomicOr(&mask[i][j >> 6], 1ull << (j & 63));
    }
    __syncthreads();
    // ---- 3. greedy scan in score order (the 2-D NMS kernel left the detections sorted by scores_3d)
    if (threadIdx.x == 0) {
        unsigned long long removed[kBevMax / 64] = {0ull, 0ull, 0ull, 0ull};
        for (int i = 0; i < n; ++i) {
            const bool r = (removed[i >> 6] >> (i & 63)) & 1ull;
            keep[i] = r ? 0 : 1;
            if (!r)
                for (int w = 0; w < kBevMax / 64; ++w) removed[w] |= mask[i][w];
        }
    }
    __syncthreads();
    // ---- 4. detector_postprocess on the survivors + order-preserving compaction (in place via registers)
    const int img_h = p.sizes[b * 4 + 0], img_w = p.sizes[b * 4 + 1], out_h = p.sizes[b * 4 + 2], out_w = p.sizes[b * 4 + 3];
    const float sxs = static_cast<float>(out_w) / static_cast<float>(img_w), sys = static_cast<float>(out_h) / static_cast<float>(img_h);
    Det mine[kBevMax / kBevThreads];
    for (int s = 0; s < kBevMax / kBevThreads; ++s) {
        const int i = threadIdx.x + s * kBevThreads;
        if (i < n) {
            mine[s] = dets[i];
            if (p.do_postprocess) {
                Det& D = mine[s];
                D.box[0] = fminf(fmaxf(D.box[0] * sxs, 0.f), static_cast<float>(out_w));
                D.box[2] = fminf(fmaxf(D.box[2] * sxs, 0.f), static_cast<float>(out_w));
                D.box[1] = fminf(fmaxf(D.box[1] * sys, 0.f), static_cast<float>(out_h));
                D.box[3] = fminf(fmaxf(D.box[3] * sys, 0.f), static_cast<float>(out_h));
                if (!((D.box[2] - D.box[0]) > 0.f && (D.box[3] - D.box[1]) > 0.f)) keep[i] = 0;
            }
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int m = 0;
        for (int i = 0; i < n; ++i) {
            new_pos[i] = m;
            m += keep[i];
        }
        s_total = m;
    }
    __syncthreads();
    for (int s = 0; s < kBevMax / kBevThreads; ++s) {
        const int i = threadIdx.x + s * kBevThreads;
        if (i < n && keep[i]) dets[new_pos[i]] = mine[s];
    }
    if (threadIdx.x == 0) p.counts[b] = s_total;
}

// One thread per pair: the rotated IoU every BEV kernel thresholds, exposed so tests can hold it to a float64 reference.
__global__ void __launch_bounds__(kBevThreads) rotated_iou_kernel(const float* a, const float* b, int n, float* out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = rotated_iou(a + static_cast<size_t>(i) * 5, b + static_cast<size_t>(i) * 5);
}

}  // namespace

cudaError_t launch_rotated_iou(const float* a, const float* b, int n, float* out, cudaStream_t stream) {
    if (n < 1) return cudaSuccess;
    rotated_iou_kernel<<<(n + kBevThreads - 1) / kBevThreads, kBevThreads, 0, stream>>>(a, b, n, out);
    return cudaGetLastError();
}

cudaError_t launch_bev_nms(Det* dets, int32_t* counts, const float* K, const float* poses, const int32_t* sizes,
                           int32_t* flags, int B, int cap, float thr, int do_postprocess, cudaStream_t stream) {
    BevParams p;
    p.dets = dets;
    p.counts = counts;
    p.K = K;
    p.poses = poses;
    p.sizes = sizes;
    p.flags = flags;
    p.cap = cap;
    p.do_postprocess = do_postprocess;
    p.thr = thr;
    bev_nms_kernel<<<B, kBevThreads, 0, stream>>>(p);
    return cudaGetLastError();
}

size_t sample_aggregate_scratch_bytes(int B, int cap) { return static_cast<size_t>(B) * cap * sizeof(float); }

cudaError_t launch_sample_aggregate(Det* dets, int32_t* counts, const float* K, const float* poses, const int32_t* group,
                                    int num_groups, float* global, void* scratch, int32_t* flags, int B, int cap,
                                    float thr, int max_dets, cudaStream_t stream) {
    if (cap > kBevMax || B >= 65536) return cudaErrorInvalidValue;
    AggParams p;
    p.dets = dets;
    p.counts = counts;
    p.K = K;
    p.poses = poses;
    p.group = group;
    p.global = global;
    p.keep_score = static_cast<float*>(scratch);
    p.flags = flags;
    p.B = B;
    p.cap = cap;
    p.max_dets = max_dets;
    p.thr = thr;
    static uint64_t configured_devices = 0;
    if (first_use_on_device(&configured_devices)) {
        const cudaError_t e = cudaFuncSetAttribute(sample_nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                   static_cast<int>(sizeof(GrpSmem)));
        if (e != cudaSuccess) return e;
    }
    sample_nms_kernel<<<num_groups, kGrpThreads, sizeof(GrpSmem), stream>>>(p);
    sample_compact_kernel<<<B, kBevThreads, 0, stream>>>(p);
    return cudaGetLastError();
}

}  // namespace dd3d
