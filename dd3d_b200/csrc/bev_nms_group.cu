// Grouped rotated BEV NMS for large detection sets, spread over the whole GPU.
//
// Serves the two BEV steps of test-time augmentation for NuscenesDD3D (nuscenes_dd3d_tta.py), whose inputs are too large
// for the one-CTA kernels of bev_nms.cu (256 boxes per image, 768 per sample group):
//   * camera mode -- bev_nms(merged_instances.pred_boxes3d, ...) on the merged set of one image (<= kTtaMergedMax boxes),
//     with the default pose_cam_global = CAMERA_TO_VEHICLE_ROTATION (tridet/layers/bev_nms.py:99-133);
//   * global mode -- nuscenes_sample_aggregate over the images of the call (postprocessing.py:22-108): boxes to the global
//     frame through each image's pose, one class-aware rotated NMS per sample group, keep[:max_dets] on the score-sorted
//     survivors of the WHOLE call, survivors split back per image in their original order, pred_boxes3d_global attached.
// Each detection's translation comes from the intrinsics of the view it was detected in (a [B][num_views][9] table indexed
// by Det::level, which the TTA merge sets to the view index): Boxes3D.from_vectors(..., orig_intrinsics) per view.
//
// Pipeline (the rotated counterpart of nms.cu's sort / mask / scan / finish):
//   layout   1 CTA        images -> groups: concatenation offsets (image order inside a group), group sizes, mask space
//   prep     B x slots    one thread per box: tvec, pose transform, BEV rectangle, pred_boxes3d_global, sort key
//   sort     1 CTA/group  bitonic sort in shared memory: class major, scores_3d descending, concatenation index
//   mask     all SMs      one warp per row of a class segment: rotated-IoU bit matrix in global scratch
//   scan     1 CTA per (group, class)   greedy pass, 64 rows at a time; survivors publish their score
//   select   1 CTA        radix select of the max_dets-th survivor key of the call (only when the cap binds)
//   compact  1 CTA/image  order-preserving compaction of dets / global rows, new counts
// Every output is written from scratch each call and no step depends on CTA scheduling order: bit-deterministic.
#include "bev_geom.cuh"
#include "device_once.cuh"
#include "pdl.cuh"

namespace dd3d {

namespace {

constexpr int kGbMaxB = 256;          // images per call
constexpr int kGbMaxCap = 1024;       // detection slots per image (kTtaMergedMax)
constexpr int kGbGroupImages = 16;    // images per group (the caller's max_group_images is at most this)
constexpr int kGbMaxCls = 64;         // class ids 0..63
constexpr int kGbSortMax = kGbGroupImages * kGbMaxCap;  // boxes per group
constexpr int kGbMaxWords = kGbSortMax / 64;
constexpr int kGbSortThreads = 1024;
constexpr int kGbThreads = 256;
constexpr int kGbPrepThreads = 128;
constexpr int kGbFlag = 32;           // capacity exceeded (a count above cap, more than max_group_images images in a
                                      // group, group, class or view index out of range)
static_assert(kGbMaxCap <= 1024, "compaction runs one thread per slot");
static_assert(kGbSortMax <= 65536, "the sort key holds the concatenation index in 16 bits");

struct GbParams {
    Det* dets;             // [B][cap], compacted in place
    int32_t* counts;       // [B]
    const float* view_K;   // [B][num_views][9] intrinsics each detection's translation is computed with
    const float* poses;    // [B][7] global camera pose (w, x, y, z, tx, ty, tz); global mode only
    const int32_t* group;  // [B]
    float* global;         // [B][cap][10] quat (w, x, y, z), tvec, size in the pose's frame, or nullptr
    int32_t* flags;
    int B, cap, num_views, pose_mode, num_groups, max_group_images, max_dets;
    float thr;
    // scratch
    int32_t* img_n;              // [B] boxes of image b that enter the NMS
    int32_t* img_pos;            // [B] concatenation index of image b's slot 0
    int32_t* grp;                // [num_groups][3] first concatenation index, size, first mask word
    int32_t* total;              // [1] boxes of the call
    unsigned long long* key;     // [N] by concatenation index: class << 48 | ~score bits << 16 | index in the group
    float* rect;                 // [N][5] by concatenation index: BEV rectangle (cx, cy, w, h, angle in degrees)
    int32_t* src;                // [N] by concatenation index: b * cap + slot
    float* srect;                // [N][5] by sorted position
    int32_t* ssrc;               // [N] by sorted position
    int4* row;                   // [N] by sorted position: segment start, segment size, first mask word, row in segment
    int4* seg;                   // [num_groups][kGbMaxCls] start, size, first mask word of each class segment
    unsigned long long* mask;    // rows of the class segments, ceil(size / 64) words each
    float* keep_score;           // [B][cap] scores_3d of the NMS survivors, -1 elsewhere
    unsigned long long* sel;     // [2] key of the max_dets-th survivor, capped
};

struct GbScratch {
    size_t img_n, img_pos, grp, total, key, rect, src, srect, ssrc, row, seg, mask, keep_score, sel, bytes;
};

size_t align256(size_t x) { return (x + 255) / 256 * 256; }

GbScratch gb_layout(int B, int cap, int max_group_images) {
    const size_t N = static_cast<size_t>(B) * cap;
    // a group of n boxes needs at most n * ceil(n / 64) mask words (sum over its class segments), n <= max_group_images * cap
    const size_t words = N * ((static_cast<size_t>(max_group_images) * cap + 63) / 64);
    GbScratch s;
    size_t o = 0;
    auto take = [&](size_t bytes) {
        const size_t at = o;
        o += align256(bytes);
        return at;
    };
    s.img_n = take(B * 4);
    s.img_pos = take(B * 4);
    s.grp = take(static_cast<size_t>(B) * 3 * 4);
    s.total = take(4);
    s.key = take(N * 8);
    s.rect = take(N * 5 * 4);
    s.src = take(N * 4);
    s.srect = take(N * 5 * 4);
    s.ssrc = take(N * 4);
    s.row = take(N * 16);
    s.seg = take(static_cast<size_t>(B) * kGbMaxCls * 16);
    s.mask = take(words * 8);
    s.keep_score = take(N * 4);
    s.sel = take(16);
    s.bytes = o;
    return s;
}

// pose_cam_global = CAMERA_TO_VEHICLE_ROTATION (bev_nms.py:27-32): x_vehicle = z_cam, y_vehicle = -x_cam, z_vehicle = -y_cam
__constant__ float kCamToVehicle[9] = {0.f, 0.f, 1.f, -1.f, 0.f, 0.f, 0.f, -1.f, 0.f};

__global__ void __launch_bounds__(32) gbev_layout_kernel(const GbParams p) {
    DD3D_PDL_PROLOGUE();
    __shared__ int s_n[kGbMaxB], s_imgs[kGbMaxB], s_local[kGbMaxB], s_base[kGbMaxB];
    if (threadIdx.x != 0) return;
    for (int g = 0; g < p.num_groups; ++g) s_n[g] = s_imgs[g] = 0;
    int bad = 0;
    for (int b = 0; b < p.B; ++b) {
        const int g = p.group[b];
        p.img_n[b] = 0;
        s_local[b] = 0;
        if (g < 0 || g >= p.num_groups || s_imgs[g] == p.max_group_images) {
            bad = 1;
            continue;
        }
        if (p.counts[b] > p.cap) bad = 1;  // fail loudly rather than truncate
        const int c = min(max(p.counts[b], 0), p.cap);
        ++s_imgs[g];
        s_local[b] = s_n[g];
        s_n[g] += c;
        p.img_n[b] = c;
    }
    int base = 0, mbase = 0;
    for (int g = 0; g < p.num_groups; ++g) {
        const int n = s_n[g];
        p.grp[g * 3 + 0] = base;
        p.grp[g * 3 + 1] = n;
        p.grp[g * 3 + 2] = mbase;
        s_base[g] = base;
        base += n;
        mbase += n * ((n + 63) / 64);
    }
    *p.total = base;
    for (int b = 0; b < p.B; ++b) {
        const int g = p.group[b];
        p.img_pos[b] = (g >= 0 && g < p.num_groups) ? s_base[g] + s_local[b] : 0;
    }
    if (bad) atomicOr(p.flags, kGbFlag);
}

__global__ void __launch_bounds__(kGbPrepThreads) gbev_prep_kernel(const GbParams p) {
    DD3D_PDL_PROLOGUE();
    const int b = blockIdx.y, s = blockIdx.x * kGbPrepThreads + threadIdx.x;
    if (s >= p.cap) return;
    const size_t flat = static_cast<size_t>(b) * p.cap + s;
    p.keep_score[flat] = -1.0f;
    if (s >= p.img_n[b]) return;
    const Det& D = p.dets[flat];
    int view = p.num_views > 1 ? D.level : 0;
    if (view < 0 || view >= p.num_views) {
        atomicOr(p.flags, kGbFlag);
        view = 0;
    }
    float iK[9], Rw[9], R[9], t[3], rect[5];
    invert_K(p.view_K + (static_cast<size_t>(b) * p.num_views + view) * 9, iK);
    const float zero[3] = {0.f, 0.f, 0.f};
    const float* pose_t = zero;
    if (p.pose_mode == 0) {
        quat_to_mat3(p.poses + b * 7, Rw);
        pose_t = p.poses + b * 7 + 4;
    } else {
#pragma unroll
        for (int i = 0; i < 9; ++i) Rw[i] = kCamToVehicle[i];
    }
    box_to_global(D, iK, Rw, pose_t, R, t, rect);
    const int concat = p.img_pos[b] + s;
#pragma unroll
    for (int i = 0; i < 5; ++i) p.rect[static_cast<size_t>(concat) * 5 + i] = rect[i];
    if (p.global) {
        float q[4];
        mat3_to_quat(R, q);
        float* go = p.global + flat * 10;
        go[0] = q[0]; go[1] = q[1]; go[2] = q[2]; go[3] = q[3];
        go[4] = t[0]; go[5] = t[1]; go[6] = t[2];
        go[7] = D.size[0]; go[8] = D.size[1]; go[9] = D.size[2];
    }
    int cls = D.cls;
    if (cls < 0 || cls >= kGbMaxCls) {
        atomicOr(p.flags, kGbFlag);
        cls = min(max(cls, 0), kGbMaxCls - 1);
    }
    const int local = concat - p.grp[p.group[b] * 3];
    // class major; descending scores_3d (non-negative floats order like their bit patterns); concatenation index
    p.key[concat] = (static_cast<unsigned long long>(cls) << 48) |
                    (static_cast<unsigned long long>(~__float_as_uint(D.score3d)) << 16) | static_cast<unsigned>(local);
    p.src[concat] = static_cast<int32_t>(flat);
}

__global__ void __launch_bounds__(kGbSortThreads) gbev_sort_kernel(const GbParams p) {
    DD3D_PDL_PROLOGUE();
    extern __shared__ __align__(16) unsigned char smem_raw[];
    unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem_raw);
    __shared__ int s_cnt[kGbMaxCls], s_start[kGbMaxCls], s_moff[kGbMaxCls];
    const int g = blockIdx.x;
    const int base = p.grp[g * 3 + 0], n = p.grp[g * 3 + 1], mbase = p.grp[g * 3 + 2];
    int n2 = 1;
    while (n2 < n) n2 <<= 1;
    for (int c = threadIdx.x; c < kGbMaxCls; c += blockDim.x) s_cnt[c] = 0;
    for (int i = threadIdx.x; i < n2; i += blockDim.x) keys[i] = i < n ? p.key[base + i] : ~0ull;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) atomicAdd(&s_cnt[static_cast<int>(keys[i] >> 48)], 1);
    for (int k = 2; k <= n2; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            __syncthreads();
            for (int i = threadIdx.x; i < n2; i += blockDim.x) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const unsigned long long a = keys[i], b2 = keys[ixj];
                    if ((a > b2) == ((i & k) == 0)) {
                        keys[i] = b2;
                        keys[ixj] = a;
                    }
                }
            }
        }
    __syncthreads();
    if (threadIdx.x == 0) {
        int start = 0, moff = mbase;
        for (int c = 0; c < kGbMaxCls; ++c) {
            const int m = s_cnt[c];
            s_start[c] = start;
            s_moff[c] = moff;
            p.seg[g * kGbMaxCls + c] = make_int4(base + start, m, moff, 0);
            start += m;
            moff += m * ((m + 63) / 64);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const unsigned long long k = keys[i];
        const int c = static_cast<int>(k >> 48);
        const size_t from = static_cast<size_t>(base) + (k & 0xffffull), to = static_cast<size_t>(base) + i;
#pragma unroll
        for (int e = 0; e < 5; ++e) p.srect[to * 5 + e] = p.rect[from * 5 + e];
        p.ssrc[to] = p.src[from];
        p.row[to] = make_int4(base + s_start[c], s_cnt[c], s_moff[c], i - s_start[c]);
    }
}

// Rectangles whose bounding circles are apart (with a relative margin far above fp32 rounding) are disjoint: their IoU is
// exactly 0 in the polygon clipper as well, so for iou_thresh >= 0 the pair never suppresses and needs no clipping.
__device__ __forceinline__ bool circles_apart(const float* a, const float* b) {
    const float ra = 0.5f * sqrtf(a[2] * a[2] + a[3] * a[3]), rb = 0.5f * sqrtf(b[2] * b[2] + b[3] * b[3]);
    const float dx = a[0] - b[0], dy = a[1] - b[1], r = (ra + rb) * 1.001f + 1e-4f;
    return dx * dx + dy * dy > r * r;
}

__global__ void __launch_bounds__(kGbThreads) gbev_mask_kernel(const GbParams p) {
    DD3D_PDL_PROLOGUE();
    const int total = *p.total;
    const int lane = threadIdx.x & 31;
    const int nwarps = gridDim.x * (kGbThreads / 32);
    const bool reject = p.thr >= 0.f;
    for (int P = blockIdx.x * (kGbThreads / 32) + (threadIdx.x >> 5); P < total; P += nwarps) {
        const int4 ri = p.row[P];
        const int start = ri.x, n = ri.y, r = ri.w, W = (n + 63) / 64;
        float a[5];
#pragma unroll
        for (int e = 0; e < 5; ++e) a[e] = p.srect[static_cast<size_t>(P) * 5 + e];
        unsigned long long* out = p.mask + static_cast<size_t>(ri.z) + static_cast<size_t>(r) * W;
        for (int w = r >> 6; w < W; ++w) {  // the scan reads a row's diagonal word and the words right of it only
            unsigned bits[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int j = w * 64 + h * 32 + lane;
                bool hit = false;
                if (j > r && j < n) {
                    float c[5];
#pragma unroll
                    for (int e = 0; e < 5; ++e) c[e] = p.srect[(static_cast<size_t>(start) + j) * 5 + e];
                    hit = !(reject && circles_apart(a, c)) && rotated_iou(a, c) > p.thr;
                }
                bits[h] = __ballot_sync(0xffffffffu, hit);
            }
            if (lane == 0) out[w] = static_cast<unsigned long long>(bits[0]) | (static_cast<unsigned long long>(bits[1]) << 32);
        }
    }
}

__global__ void __launch_bounds__(kGbThreads) gbev_scan_kernel(const GbParams p) {
    DD3D_PDL_PROLOGUE();
    __shared__ unsigned long long removed[kGbMaxWords];
    __shared__ unsigned long long diag[64];
    __shared__ unsigned long long s_kept;
    const int4 sg = p.seg[blockIdx.x * kGbMaxCls + blockIdx.y];
    const int start = sg.x, n = sg.y;
    if (n == 0) return;
    const int W = (n + 63) / 64;
    const unsigned long long* mask = p.mask + static_cast<size_t>(sg.z);
    for (int w = threadIdx.x; w < W; w += blockDim.x) removed[w] = 0ull;
    __syncthreads();
    for (int rb = 0; rb < W; ++rb) {
        const int rows = min(64, n - rb * 64);
        if (threadIdx.x < rows) diag[threadIdx.x] = mask[static_cast<size_t>(rb * 64 + threadIdx.x) * W + rb];
        __syncthreads();
        if (threadIdx.x == 0) {  // greedy inside the 64-row block
            unsigned long long rem = removed[rb], kept = 0ull;
            for (int i = 0; i < rows; ++i)
                if (!((rem >> i) & 1ull)) {
                    kept |= 1ull << i;
                    rem |= diag[i];
                }
            s_kept = kept;
        }
        __syncthreads();
        const unsigned long long kept = s_kept;
        for (int w = rb + 1 + threadIdx.x; w < W; w += blockDim.x) {  // the block's survivors suppress later rows
            unsigned long long acc = removed[w];
            for (unsigned long long k = kept; k; k &= k - 1)
                acc |= mask[static_cast<size_t>(rb * 64 + __ffsll(static_cast<long long>(k)) - 1) * W + w];
            removed[w] = acc;
        }
        if (threadIdx.x < rows && ((kept >> threadIdx.x) & 1ull)) {
            const int flat = p.ssrc[start + rb * 64 + threadIdx.x];
            p.keep_score[flat] = p.dets[flat].score3d;
        }
        __syncthreads();
    }
}

// key of a survivor in the NMS output order of the whole call: scores_3d descending, then image, then slot
__device__ __forceinline__ unsigned long long survivor_key(float score, size_t flat) {
    return (static_cast<unsigned long long>(~__float_as_uint(score)) << 32) | static_cast<unsigned long long>(flat);
}

__global__ void __launch_bounds__(kGbSortThreads) gbev_select_kernel(const GbParams p) {
    DD3D_PDL_PROLOGUE();
    __shared__ unsigned s_hist[256];
    __shared__ int s_total, s_k;
    __shared__ unsigned long long s_prefix;
    const size_t N = static_cast<size_t>(p.B) * p.cap;
    if (threadIdx.x == 0) s_total = 0;
    __syncthreads();
    int part = 0;
    for (size_t i = threadIdx.x; i < N; i += blockDim.x) part += p.keep_score[i] >= 0.f;
    atomicAdd(&s_total, part);
    __syncthreads();
    if (p.max_dets <= 0 || s_total <= p.max_dets) {
        if (threadIdx.x == 0) {
            p.sel[0] = ~0ull;
            p.sel[1] = 0ull;
        }
        return;
    }
    if (threadIdx.x == 0) {
        s_k = p.max_dets;  // 1-based rank of the last survivor kept
        s_prefix = 0ull;
    }
    // radix select, 8 bits at a time from the top: the keys are unique, so "key <= k-th key" keeps exactly max_dets
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (int d = threadIdx.x; d < 256; d += blockDim.x) s_hist[d] = 0u;
        __syncthreads();
        const unsigned long long prefix = s_prefix;
        const unsigned long long high = shift == 56 ? 0ull : (~0ull << (shift + 8));
        for (size_t i = threadIdx.x; i < N; i += blockDim.x) {
            const float sc = p.keep_score[i];
            if (sc < 0.f) continue;
            const unsigned long long k = survivor_key(sc, i);
            if ((k & high) == prefix) atomicAdd(&s_hist[(k >> shift) & 255ull], 1u);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            int cum = 0;
            for (int d = 0; d < 256; ++d) {
                if (cum + static_cast<int>(s_hist[d]) >= s_k) {
                    s_prefix = prefix | (static_cast<unsigned long long>(d) << shift);
                    s_k -= cum;
                    break;
                }
                cum += s_hist[d];
            }
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        p.sel[0] = s_prefix;
        p.sel[1] = 1ull;
    }
}

__global__ void __launch_bounds__(kGbMaxCap) gbev_compact_kernel(const GbParams p) {
    DD3D_PDL_PROLOGUE();
    __shared__ int s_warp[kGbMaxCap / 32];
    const int b = blockIdx.x, s = threadIdx.x, lane = s & 31, warp = s >> 5;
    const size_t flat = static_cast<size_t>(b) * p.cap + s;
    const bool capped = p.sel[1] != 0ull;
    const unsigned long long last = p.sel[0];
    bool keep = false;
    Det d;
    float gl[10];
    if (s < p.cap) {
        const float sc = p.keep_score[flat];
        keep = sc >= 0.f && (!capped || survivor_key(sc, flat) <= last);
        if (keep) {
            d = p.dets[flat];
            if (p.global)
#pragma unroll
                for (int e = 0; e < 10; ++e) gl[e] = p.global[flat * 10 + e];
        }
    }
    const unsigned ballot = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) s_warp[warp] = __popc(ballot);
    __syncthreads();  // every read of this image's slots happened above
    int off = 0;
    for (int w = 0; w < warp; ++w) off += s_warp[w];
    if (keep) {
        const size_t to = static_cast<size_t>(b) * p.cap + off + __popc(ballot & ((1u << lane) - 1u));
        p.dets[to] = d;
        if (p.global)
#pragma unroll
            for (int e = 0; e < 10; ++e) p.global[to * 10 + e] = gl[e];
    }
    if (s == 0) {
        int total = 0;
        for (int w = 0; w < static_cast<int>(blockDim.x) / 32; ++w) total += s_warp[w];
        p.counts[b] = total;
    }
}

}  // namespace

size_t group_bev_nms_scratch_bytes(int B, int cap, int max_group_images) {
    if (B < 1 || cap < 1 || max_group_images < 1) return 0;
    return gb_layout(B, cap, max_group_images).bytes;
}

cudaError_t launch_group_bev_nms(Det* dets, int32_t* counts, const float* view_K, int num_views, const float* poses,
                                 int pose_mode, const int32_t* group, int num_groups, int max_group_images, float* global,
                                 void* scratch, int32_t* flags, int B, int cap, float thr, int max_dets,
                                 cudaStream_t stream) {
    if (B < 1 || B > kGbMaxB || cap < 1 || cap > kGbMaxCap || num_groups < 1 || num_groups > B || num_views < 1 ||
        max_group_images < 1 || max_group_images > kGbGroupImages ||
        (pose_mode != 0 && pose_mode != 1) || (pose_mode == 0 && poses == nullptr))
        return cudaErrorInvalidValue;
    const GbScratch L = gb_layout(B, cap, max_group_images);
    uint8_t* s = static_cast<uint8_t*>(scratch);
    GbParams p;
    p.dets = dets;
    p.counts = counts;
    p.view_K = view_K;
    p.poses = poses;
    p.group = group;
    p.global = global;
    p.flags = flags;
    p.B = B;
    p.cap = cap;
    p.num_views = num_views;
    p.pose_mode = pose_mode;
    p.num_groups = num_groups;
    p.max_group_images = max_group_images;
    p.max_dets = max_dets;
    p.thr = thr;
    p.img_n = reinterpret_cast<int32_t*>(s + L.img_n);
    p.img_pos = reinterpret_cast<int32_t*>(s + L.img_pos);
    p.grp = reinterpret_cast<int32_t*>(s + L.grp);
    p.total = reinterpret_cast<int32_t*>(s + L.total);
    p.key = reinterpret_cast<unsigned long long*>(s + L.key);
    p.rect = reinterpret_cast<float*>(s + L.rect);
    p.src = reinterpret_cast<int32_t*>(s + L.src);
    p.srect = reinterpret_cast<float*>(s + L.srect);
    p.ssrc = reinterpret_cast<int32_t*>(s + L.ssrc);
    p.row = reinterpret_cast<int4*>(s + L.row);
    p.seg = reinterpret_cast<int4*>(s + L.seg);
    p.mask = reinterpret_cast<unsigned long long*>(s + L.mask);
    p.keep_score = reinterpret_cast<float*>(s + L.keep_score);
    p.sel = reinterpret_cast<unsigned long long*>(s + L.sel);
    const size_t sort_smem = static_cast<size_t>(kGbSortMax) * sizeof(unsigned long long);
    static uint64_t configured_devices = 0;
    if (first_use_on_device(&configured_devices)) {
        const cudaError_t e = cudaFuncSetAttribute(gbev_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                   static_cast<int>(sort_smem));
        if (e != cudaSuccess) return e;
    }
    int dev = 0, sms = 132;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaError_t e = launch_pdl(gbev_layout_kernel, dim3(1), dim3(32), 0, stream, p);
    if (e == cudaSuccess)
        e = launch_pdl(gbev_prep_kernel, dim3((cap + kGbPrepThreads - 1) / kGbPrepThreads, B), dim3(kGbPrepThreads), 0,
                       stream, p);
    if (e == cudaSuccess) e = launch_pdl(gbev_sort_kernel, dim3(num_groups), dim3(kGbSortThreads), sort_smem, stream, p);
    if (e == cudaSuccess) e = launch_pdl(gbev_mask_kernel, dim3(sms * 8), dim3(kGbThreads), 0, stream, p);
    if (e == cudaSuccess) e = launch_pdl(gbev_scan_kernel, dim3(num_groups, kGbMaxCls), dim3(kGbThreads), 0, stream, p);
    if (e == cudaSuccess) e = launch_pdl(gbev_select_kernel, dim3(1), dim3(kGbSortThreads), 0, stream, p);
    if (e == cudaSuccess)
        e = launch_pdl(gbev_compact_kernel, dim3(B), dim3((cap + 31) / 32 * 32), 0, stream, p);
    return e;
}

}  // namespace dd3d
