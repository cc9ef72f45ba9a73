// Per-image class-aware greedy NMS + post-NMS top-k + rescale/clip, no host sync.
//
// Replaces Instances.cat over levels + FCOS2DInference.nms_and_top_k (reference core.py:130-135, fcos2d.py:346-367
// -> detectron2 batched_nms -> torchvision nms) and detectron2 detector_postprocess (core.py:153-160):
//   1. gather the <= L*topk decoded candidates of the image, order them by (score_3d desc, level asc, index asc)
//      (deterministic regardless of the atomics order upstream);
//   2. greedy NMS in that order (IoU > thr, same class => suppressed; IoU = inter / (a + b - inter) exactly as torchvision);
//   3. if more than POST_NMS_TOPK remain keep those whose 2-D score >= the k-th largest 2-D score (fcos2d.py:359-365);
//   4. scale boxes to the requested output size, clip, drop empty boxes (detector_postprocess).
// Two forms with identical results: `nms_kernel`, one CTA per image doing all four steps (in-smem bitonic sort, 64 boxes per
// greedy step) -- the TTA merge and DO_NMS = False use it; and the engine's default multi-CTA path further down
// (rank sort -> IoU bit matrix -> per-class scan -> finish), which keeps all SMs busy when one class holds most candidates.
#include "detect.cuh"
#include "device_once.cuh"
#include "pdl.cuh"

#include <stdlib.h>

namespace dd3d {

namespace {

constexpr int kNmsThreads = 1024;
constexpr int kMaxCand = kNmsSortCap;  // bitonic sort capacity (>= L * topk)

// ascending bitonic sort of n2 (power of two) 64-bit keys with a 16-bit payload, in shared memory
__device__ void bitonic_sort(uint64_t* key, uint16_t* val, int n2) {
    for (int k = 2; k <= n2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < n2; i += blockDim.x) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const uint64_t a = key[i], b = key[ixj];
                    const bool up = ((i & k) == 0);
                    if ((a > b) == up) {
                        key[i] = b;
                        key[ixj] = a;
                        const uint16_t t = val[i];
                        val[i] = val[ixj];
                        val[ixj] = t;
                    }
                }
            }
            __syncthreads();
        }
    }
}

// order-preserving compaction: dst gets the indices i (0..n) with flag[i] != 0; returns the count
__device__ int compact_indices(const uint8_t* flag, int n, int* dst, int* s_warp_sums, int* s_base) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) *s_base = 0;
    __syncthreads();
    for (int start = 0; start < n; start += blockDim.x) {
        const int i = start + threadIdx.x;
        const int f = (i < n && flag[i]) ? 1 : 0;
        const unsigned m = __ballot_sync(0xffffffffu, f);
        const int prefix = __popc(m & ((1u << lane) - 1));
        if (lane == 0) s_warp_sums[warp] = __popc(m);
        __syncthreads();
        if (warp == 0) {
            int v = s_warp_sums[lane];
            int incl = v;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += t;
            }
            s_warp_sums[lane] = incl - v;  // exclusive
            if (lane == 31) s_warp_sums[32] = incl;
        }
        __syncthreads();
        const int base = *s_base;
        if (f) dst[base + s_warp_sums[warp] + prefix] = i;
        __syncthreads();
        if (threadIdx.x == 0) *s_base = base + s_warp_sums[32];
        __syncthreads();
    }
    return *s_base;
}

// ---------------------------------------------------------------------------------------------- building blocks
// Shared-memory working set of one image (cap = L * topk candidates).
struct NmsSmem {
    uint64_t* key;   // [kMaxCand]
    float4* boxes;   // [cap]
    int* list;       // [cap]
    int* list2;      // [cap]
    uint16_t* val;   // [kMaxCand]  sorted position -> candidate slot
    uint8_t* cls;    // [cap]
    uint8_t* flag;   // [cap]
};

__device__ __forceinline__ NmsSmem carve(uint8_t* raw, int cap) {
    NmsSmem m;
    m.key = reinterpret_cast<uint64_t*>(raw);
    m.boxes = reinterpret_cast<float4*>(m.key + kMaxCand);
    m.list = reinterpret_cast<int*>(m.boxes + cap);
    m.list2 = m.list + cap;
    m.val = reinterpret_cast<uint16_t*>(m.list2 + cap);
    m.cls = reinterpret_cast<uint8_t*>(m.val + kMaxCand);
    m.flag = m.cls + cap;
    return m;
}

// 1. keys (score3d desc, level asc, index asc) -> bitonic sort (when do_nms) -> val[i] = candidate slot of sorted position i.
//    Returns n.  s_lvl_off: [kLevels + 1] shared ints; positions num_levels and up are empty.
__device__ int sort_candidates(const NmsParams& p, int b, const Det* cand, NmsSmem m, int* s_lvl_off) {
    if (threadIdx.x == 0) {
        int off = 0;
        for (int l = 0; l < kLevels; ++l) {
            s_lvl_off[l] = off;
            if (l < p.num_levels) off += min(p.cand_count[b * p.num_levels + l], p.topk);
        }
        s_lvl_off[kLevels] = off;
    }
    __syncthreads();
    const int n = s_lvl_off[kLevels];
    int n2 = 1;
    while (n2 < n) n2 <<= 1;
    for (int i = threadIdx.x; i < n2; i += blockDim.x) {
        uint64_t k = ~0ull;
        uint16_t v = 0;
        if (i < n) {
            int l = 0;
#pragma unroll
            for (int t = 1; t < kLevels; ++t)
                if (i >= s_lvl_off[t]) l = t;
            const int slot = l * p.topk + (i - s_lvl_off[l]);
            const Det& d = cand[slot];
            const uint32_t sb = ~__float_as_uint(d.score3d);  // positive floats: larger score -> smaller key
            k = (static_cast<uint64_t>(sb) << 32) | (static_cast<uint64_t>(l) << 28) | static_cast<uint32_t>(d.index);
            v = static_cast<uint16_t>(slot);
        }
        m.key[i] = k;
        m.val[i] = v;
    }
    __syncthreads();
    if (p.do_nms) bitonic_sort(m.key, m.val, n2);
    return n;
}

// 2. greedy NMS over n boxes already in score order, 64 boxes per step: resolve the 64x64 diagonal block serially (warp 0),
//    then let all threads test the remaining boxes against the step's survivors.  cls == nullptr: single class.
//    flag[i] = 1 where removed (must be 0 on entry).  blockDim.x must be a multiple of 64 and >= 64.
__device__ void greedy_nms(const float4* boxes, const uint8_t* cls, uint8_t* flag, int n, float thr,
                           unsigned long long* s_diag, unsigned long long* s_kept_mask) {
    const int tpr = blockDim.x >> 6;  // threads per row of the diagonal block
    const int cpt = 64 / tpr;         // columns per thread
    for (int c0 = 0; c0 < n; c0 += 64) {
        const int cn = min(64, n - c0);
        {
            const int i = threadIdx.x / tpr, part = threadIdx.x - i * tpr;
            unsigned long long m = 0ull;
            if (i < cn) {
                const float4 bi = boxes[c0 + i];
                const int ci = cls ? cls[c0 + i] : 0;
                for (int u = 0; u < cpt; ++u) {
                    const int j = part * cpt + u;
                    if (j > i && j < cn && (cls == nullptr || cls[c0 + j] == ci) && iou_tv(bi, boxes[c0 + j]) > thr) m |= 1ull << j;
                }
            }
            for (int o = 1; o < tpr; o <<= 1) m |= __shfl_xor_sync(0xffffffffu, m, o);  // tpr is a power of two <= 32
            if (part == 0) s_diag[i] = m;
        }
        __syncthreads();
        if (threadIdx.x < 32) {
            const int l = threadIdx.x;
            const unsigned long long d_lo = s_diag[l], d_hi = s_diag[l + 32];
            const unsigned r_lo = __ballot_sync(0xffffffffu, l < cn && flag[c0 + l]);
            const unsigned r_hi = __ballot_sync(0xffffffffu, l + 32 < cn && flag[c0 + l + 32]);
            unsigned long long removed = (static_cast<unsigned long long>(r_hi) << 32) | r_lo;
            if (cn < 64) removed |= ~0ull << cn;
            unsigned long long kept = 0ull;
#pragma unroll 8
            for (int i = 0; i < 64; ++i) {
                const unsigned long long di = __shfl_sync(0xffffffffu, i < 32 ? d_lo : d_hi, i & 31);
                if (!((removed >> i) & 1ull)) {
                    kept |= 1ull << i;
                    removed |= di;
                }
            }
            if (l == 0) *s_kept_mask = kept;
            if (l < cn) flag[c0 + l] = ((kept >> l) & 1ull) ? 0 : 1;
            if (l + 32 < cn) flag[c0 + l + 32] = ((kept >> (l + 32)) & 1ull) ? 0 : 1;
        }
        __syncthreads();
        const unsigned long long kept = *s_kept_mask;
        for (int k = c0 + cn + threadIdx.x; k < n; k += blockDim.x) {
            if (flag[k]) continue;
            const float4 bk = boxes[k];
            const int ck = cls ? cls[k] : 0;
            unsigned long long m = kept;
            bool rem = false;
            while (m) {
                const int i = __ffsll(static_cast<long long>(m)) - 1;
                m &= m - 1;
                if ((cls == nullptr || cls[c0 + i] == ck) && iou_tv(boxes[c0 + i], bk) > thr) {
                    rem = true;
                    break;
                }
            }
            if (rem) flag[k] = 1;
        }
        __syncthreads();
    }
}

// 3. + 4. survivors (flag[i] = 1 where KEPT, sorted order) -> post-NMS top-k on the 2-D score -> detector_postprocess -> out
__device__ void finish_image(const NmsParams& p, int b, const Det* cand, NmsSmem m, int n, bool have_keep_flags,
                             int* s_warp_sums, int* s_base) {
    int nkeep = n;
    if (have_keep_flags) {
        nkeep = compact_indices(m.flag, n, m.list, s_warp_sums, s_base);
    } else {
        for (int i = threadIdx.x; i < n; i += blockDim.x) m.list[i] = i;
        __syncthreads();
    }
    // ---- post-NMS top-k on the 2-D score (>= k-th value keeps ties)
    if (p.do_nms && p.post_topk > 0 && nkeep > p.post_topk) {
        int m2 = 1;
        while (m2 < nkeep) m2 <<= 1;
        uint16_t* dummy = reinterpret_cast<uint16_t*>(m.list2);  // payload not needed; reuse list2 as scratch
        for (int i = threadIdx.x; i < m2; i += blockDim.x) {
            uint64_t k = ~0ull;
            if (i < nkeep) k = static_cast<uint64_t>(~__float_as_uint(cand[m.val[m.list[i]]].score));
            m.key[i] = k;
            dummy[i] = 0;
        }
        __syncthreads();
        // NOTE: sorting `key` destroys the sort keys of step 1 (no longer needed); val[] must stay intact,
        // so the payload array handed to the sort is the scratch one.
        bitonic_sort(m.key, dummy, m2);
        const uint32_t thr_bits = ~static_cast<uint32_t>(m.key[p.post_topk - 1]);
        const float thr = __uint_as_float(thr_bits);
        for (int i = threadIdx.x; i < nkeep; i += blockDim.x) m.flag[i] = (cand[m.val[m.list[i]]].score >= thr) ? 1 : 0;
        __syncthreads();
        const int k2 = compact_indices(m.flag, nkeep, m.list2, s_warp_sums, s_base);
        for (int i = threadIdx.x; i < k2; i += blockDim.x) m.list2[i] = m.list[m.list2[i]];
        __syncthreads();
        for (int i = threadIdx.x; i < k2; i += blockDim.x) m.list[i] = m.list2[i];
        __syncthreads();
        nkeep = k2;
    }
    // ---- detector_postprocess: scale, clip, drop empty
    const int img_h = p.sizes[b * 4 + 0], img_w = p.sizes[b * 4 + 1];
    const int out_h = p.sizes[b * 4 + 2], out_w = p.sizes[b * 4 + 3];
    const float sx = static_cast<float>(out_w) / static_cast<float>(img_w);
    const float sy = static_cast<float>(out_h) / static_cast<float>(img_h);
    if (p.do_postprocess) {
        for (int i = threadIdx.x; i < nkeep; i += blockDim.x) {
            float4 bx = m.boxes[m.list[i]];
            bx.x = fminf(fmaxf(bx.x * sx, 0.f), static_cast<float>(out_w));
            bx.z = fminf(fmaxf(bx.z * sx, 0.f), static_cast<float>(out_w));
            bx.y = fminf(fmaxf(bx.y * sy, 0.f), static_cast<float>(out_h));
            bx.w = fminf(fmaxf(bx.w * sy, 0.f), static_cast<float>(out_h));
            m.flag[i] = ((bx.z - bx.x) > 0.f && (bx.w - bx.y) > 0.f) ? 1 : 0;
        }
        __syncthreads();
        const int k2 = compact_indices(m.flag, nkeep, m.list2, s_warp_sums, s_base);
        for (int i = threadIdx.x; i < k2; i += blockDim.x) m.list2[i] = m.list[m.list2[i]];
        __syncthreads();
        for (int i = threadIdx.x; i < k2; i += blockDim.x) m.list[i] = m.list2[i];
        __syncthreads();
        nkeep = k2;
    }
    if (threadIdx.x == 0) {
        if (nkeep > p.out_cap) atomicOr(p.flags, 2);
        p.out_count[b] = min(nkeep, p.out_cap);
    }
    const int nout = min(nkeep, p.out_cap);
    Det* out = p.out + static_cast<size_t>(b) * p.out_cap;
    for (int i = threadIdx.x; i < nout; i += blockDim.x) {
        Det d = cand[m.val[m.list[i]]];
        if (p.do_postprocess) {
            d.box[0] = fminf(fmaxf(d.box[0] * sx, 0.f), static_cast<float>(out_w));
            d.box[2] = fminf(fmaxf(d.box[2] * sx, 0.f), static_cast<float>(out_w));
            d.box[1] = fminf(fmaxf(d.box[1] * sy, 0.f), static_cast<float>(out_h));
            d.box[3] = fminf(fmaxf(d.box[3] * sy, 0.f), static_cast<float>(out_h));
        }
        out[i] = d;
    }
}

// ---------------------------------------------------------------------------------------------- single-CTA kernel
// One CTA per image does everything (used when no scratch is given -- the TTA merge -- and when NMS is off).
__global__ void __launch_bounds__(kNmsThreads, 1) nms_kernel(const __grid_constant__ NmsParams p) {
    DD3D_PDL_PROLOGUE();
    extern __shared__ uint8_t smem_raw[];
    const int b = blockIdx.x;
    const int cap = p.num_levels * p.topk;
    NmsSmem m = carve(smem_raw, cap);
    __shared__ int s_warp_sums[33];
    __shared__ int s_base;
    __shared__ int s_lvl_off[kLevels + 1];
    __shared__ unsigned long long s_kept_mask;
    __shared__ unsigned long long s_diag[64];
    const Det* cand = p.cand + static_cast<size_t>(b) * cap;
    const int n = sort_candidates(p, b, cand, m, s_lvl_off);
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const Det& d = cand[m.val[i]];
        m.boxes[i] = make_float4(d.box[0], d.box[1], d.box[2], d.box[3]);
        m.cls[i] = static_cast<uint8_t>(d.cls);
        m.flag[i] = 0;  // removed flag
    }
    __syncthreads();
    const bool suppress = p.do_nms && p.nms_thresh > 0.f;
    if (suppress) {
        greedy_nms(m.boxes, m.cls, m.flag, n, p.nms_thresh, s_diag, &s_kept_mask);
        for (int i = threadIdx.x; i < n; i += blockDim.x) m.flag[i] = m.flag[i] ? 0 : 1;  // keep flags = !removed
        __syncthreads();
    }
    finish_image(p, b, cand, m, n, suppress, s_warp_sums, &s_base);
}

// ---------------------------------------------------------------------------------------------- multi-CTA path
// batched_nms never lets boxes of different classes suppress each other (detectron2 batched_nms -> torchvision: per-class
// coordinate offsets), so the greedy scan is independent per (image, class) -- but one class can hold most of an image's
// candidates (the DLA-34 bench batch: 616 of 623 in one class), and the n^2 / 2 IoUs of a 600-box class would run on
// ONE SM.  Four launches:
//   nms_sort_kernel  (32 x B CTAs)       : rank sort of the image's candidates by score_3d; publish order / class and a
//                                          CLASS-MAJOR copy (boxes + sorted position, score order inside a class, 64-aligned)
//   nms_mask_kernel  (64 x B CTAs)       : IoU bit matrix of every class segment, 64 x 64 boxes per step, on all SMs
//   nms_scan_kernel  (C x B CTAs)        : the serial greedy pass over the bit matrix only (no IoU): resolve the 64 x 64
//                                          diagonal word by word, OR the survivors' rows into the removed bit vector
//   nms_finish_kernel(B CTAs)            : survivors in sorted order -> post-NMS top-k -> postprocess -> output
// Same kept set and order as the single-CTA kernel (tests/test_kernels_gpu.py compares both with the oracle).
struct NmsScratch {
    uint16_t* order;   // [B][cap] sorted position -> candidate slot
    uint8_t* cls;      // [B][cap]
    uint8_t* removed;  // [B][cap]
    int32_t* n;        // [B]
    int32_t* seg_blk;  // [B][C + 1] first 64-row block of class c in the class-major list ([C] = total blocks)
    int32_t* seg_cnt;  // [B][C] boxes of class c
    uint16_t* cpos;    // [B][capP] class-major row -> sorted position
    float4* cbox;      // [B][capP] class-major row -> box
    unsigned long long* mask;  // [B][capP][W] bit j of word w of row i: box 64 w + j of the same class (j > i) has IoU > thr
    int capP, W;
};

__host__ __device__ __forceinline__ size_t up256(size_t v) { return (v + 255) / 256 * 256; }

__host__ __device__ __forceinline__ NmsScratch bind_nms_scratch(void* scratch, int B, int cap, int C) {
    NmsScratch s;
    s.W = (cap + 63) / 64;
    s.capP = 64 * (s.W + C);
    uint8_t* q = static_cast<uint8_t*>(scratch);
    s.order = reinterpret_cast<uint16_t*>(q);
    q += up256(static_cast<size_t>(B) * cap * 2);
    s.cls = q;
    q += up256(static_cast<size_t>(B) * cap);
    s.removed = q;
    q += up256(static_cast<size_t>(B) * cap);
    s.n = reinterpret_cast<int32_t*>(q);
    q += up256(static_cast<size_t>(B) * 4);
    s.seg_blk = reinterpret_cast<int32_t*>(q);
    q += up256(static_cast<size_t>(B) * (C + 1) * 4);
    s.seg_cnt = reinterpret_cast<int32_t*>(q);
    q += up256(static_cast<size_t>(B) * C * 4);
    s.cpos = reinterpret_cast<uint16_t*>(q);
    q += up256(static_cast<size_t>(B) * s.capP * 2);
    s.cbox = reinterpret_cast<float4*>(q);
    q += up256(static_cast<size_t>(B) * s.capP * 16);
    s.mask = reinterpret_cast<unsigned long long*>(q);
    return s;
}

constexpr int kSortThreads = 256, kSortCtasPerImage = 32;

// Rank sort.  The keys (score_3d desc, level asc, index asc) are unique, so the sorted position of a candidate is the number
// of smaller keys -- n^2 independent comparisons that spread over kSortCtasPerImage CTAs per image (64 candidates per CTA
// step, four threads per candidate) instead of the 55 - 91 barrier-separated passes of a one-CTA bitonic sort (22 - 46 us).
// The same loop counts the smaller keys OF THE SAME CLASS: the candidate's row in the class-major copy (score order inside a
// class, 64-aligned class segments) that the bit-matrix kernels work on.  Every CTA rebuilds the key table and the class
// histogram itself (n <= 8192 candidates, three words each); no cross-CTA dependency, no atomics on results.
__global__ void __launch_bounds__(kSortThreads) nms_sort_kernel(const __grid_constant__ NmsParams p) {
    DD3D_PDL_PROLOGUE();
    extern __shared__ __align__(16) uint8_t smem_raw[];
    const int b = blockIdx.y;
    const int cap = p.num_levels * p.topk, C = p.num_classes;
    uint64_t* keys = reinterpret_cast<uint64_t*>(smem_raw);       // [cap]
    uint16_t* slots = reinterpret_cast<uint16_t*>(keys + cap);    // [cap]
    uint8_t* scls = reinterpret_cast<uint8_t*>(slots + cap);      // [cap]
    __shared__ int s_lvl_off[kLevels + 1];
    __shared__ int s_cnt[256], s_seg[257];
    const Det* cand = p.cand + static_cast<size_t>(b) * cap;
    const NmsScratch sc = bind_nms_scratch(p.scratch, p.B, cap, C);
    if (threadIdx.x == 0) {
        int off = 0;
        for (int l = 0; l < kLevels; ++l) {
            s_lvl_off[l] = off;
            if (l < p.num_levels) off += min(p.cand_count[b * p.num_levels + l], p.topk);
        }
        s_lvl_off[kLevels] = off;
    }
    for (int c = threadIdx.x; c < C; c += blockDim.x) s_cnt[c] = 0;
    __syncthreads();
    const int n = s_lvl_off[kLevels];
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        int l = 0;
#pragma unroll
        for (int t = 1; t < kLevels; ++t)
            if (i >= s_lvl_off[t]) l = t;
        const int slot = l * p.topk + (i - s_lvl_off[l]);
        const Det& d = cand[slot];
        const uint32_t sb = ~__float_as_uint(d.score3d);  // positive floats: larger score -> smaller key
        keys[i] = (static_cast<uint64_t>(sb) << 32) | (static_cast<uint64_t>(l) << 28) | static_cast<uint32_t>(d.index);
        slots[i] = static_cast<uint16_t>(slot);
        scls[i] = static_cast<uint8_t>(d.cls);
        atomicAdd(&s_cnt[d.cls], 1);  // a count: independent of the order of the atomics
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int blk = 0;
        for (int c = 0; c < C; ++c) {
            s_seg[c] = blk;
            blk += (s_cnt[c] + 63) >> 6;
        }
        s_seg[C] = blk;
    }
    __syncthreads();
    if (blockIdx.x == 0) {
        if (threadIdx.x == 0) sc.n[b] = n;
        for (int c = threadIdx.x; c <= C; c += blockDim.x) {
            sc.seg_blk[b * (C + 1) + c] = s_seg[c];
            if (c < C) sc.seg_cnt[b * C + c] = s_cnt[c];
        }
    }
    const int e = threadIdx.x >> 2, part = threadIdx.x & 3;
    for (int grp = blockIdx.x; grp * 64 < n; grp += gridDim.x) {
        const int i = grp * 64 + e;
        const uint64_t ki = i < n ? keys[i] : 0ull;
        const int ci = i < n ? scls[i] : 255;  // class ids are < 255
        int r = 0, rc = 0;
        for (int j = part; j < n; j += 4) {
            const int lt = keys[j] < ki ? 1 : 0;
            r += lt;
            rc += (scls[j] == ci) ? lt : 0;
        }
        r += __shfl_xor_sync(0xffffffffu, r, 1);
        r += __shfl_xor_sync(0xffffffffu, r, 2);
        rc += __shfl_xor_sync(0xffffffffu, rc, 1);
        rc += __shfl_xor_sync(0xffffffffu, rc, 2);
        if (part == 0 && i < n) {
            const int slot = slots[i];
            const size_t o = static_cast<size_t>(b) * cap + r;
            sc.order[o] = static_cast<uint16_t>(slot);
            sc.cls[o] = static_cast<uint8_t>(ci);
            sc.removed[o] = 0;
            const size_t row = static_cast<size_t>(b) * sc.capP + static_cast<size_t>(s_seg[ci]) * 64 + rc;
            const Det& d = cand[slot];
            sc.cpos[row] = static_cast<uint16_t>(r);
            sc.cbox[row] = make_float4(d.box[0], d.box[1], d.box[2], d.box[3]);
        }
    }
}

constexpr int kMaskThreads = 256;
constexpr int kMaskCtasPerImage = 64;

// IoU bit matrix.  kMaskCtasPerImage CTAs per image stride over the image's (row block, column block) pairs -- the upper
// triangles of all class segments, enumerated class by class -- so the n^2 / 2 IoUs of a large class spread over many SMs
// instead of sitting in one CTA's serial loops.  One pair = 64 x 64 boxes: thread = (row, quarter of the columns), the four
// 16-bit quarters of a word are merged with two shuffles.
__global__ void __launch_bounds__(kMaskThreads) nms_mask_kernel(const __grid_constant__ NmsParams p) {
    DD3D_PDL_PROLOGUE();
    const int b = blockIdx.y;
    const int cap = p.num_levels * p.topk, C = p.num_classes;
    const NmsScratch sc = bind_nms_scratch(p.scratch, p.B, cap, C);
    __shared__ int s_first[257];  // first pair index of class c
    __shared__ float4 s_col[64];
    const int32_t* seg = sc.seg_blk + b * (C + 1);
    const int32_t* cnt = sc.seg_cnt + b * C;
    if (threadIdx.x == 0) {
        int tot = 0;
        for (int c = 0; c < C; ++c) {
            s_first[c] = tot;
            const int nc = cnt[c], nb = (nc + 63) >> 6;
            if (nc > 1) tot += nb * (nb + 1) / 2;
        }
        s_first[C] = tot;
    }
    __syncthreads();
    const int total = s_first[C];
    const int r_in = threadIdx.x >> 2, part = threadIdx.x & 3;
    for (int q = blockIdx.x; q < total; q += gridDim.x) {
        int c = 0;
        while (s_first[c + 1] <= q) ++c;  // classes without pairs have s_first[c + 1] == s_first[c] and are skipped
        const int nc = cnt[c], nb = (nc + 63) >> 6;
        int local = q - s_first[c], rb = 0;
        while (local >= nb - rb) {
            local -= nb - rb;
            ++rb;
        }
        const int cb = rb + local;
        const size_t row0 = static_cast<size_t>(b) * sc.capP + static_cast<size_t>(seg[c]) * 64;
        const float4* boxes = sc.cbox + row0;
        __syncthreads();  // the previous pair's readers of s_col are done
        if (threadIdx.x < 64) s_col[threadIdx.x] = boxes[min(cb * 64 + threadIdx.x, nc - 1)];
        __syncthreads();
        const int row = rb * 64 + r_in;
        const float4 bi = boxes[min(row, nc - 1)];
        unsigned m16 = 0u;
#pragma unroll 4
        for (int k = 0; k < 16; ++k) {
            const int j = 16 * part + k, col = cb * 64 + j;
            if (col < nc && col > row && iou_tv(bi, s_col[j]) > p.nms_thresh) m16 |= 1u << k;
        }
        unsigned long long word = static_cast<unsigned long long>(m16) << (16 * part);
        word |= __shfl_xor_sync(0xffffffffu, word, 1);
        word |= __shfl_xor_sync(0xffffffffu, word, 2);
        if (part == 0 && row < nc) sc.mask[(row0 + row) * sc.W + cb] = word;
    }
}

constexpr int kScanThreads = 128;  // >= W (cap <= 8192)

// The serial part of the greedy NMS of one (class, image), on the bit matrix only.  Per 64-box block: the diagonal words
// (prefetched during the previous block) are resolved by one thread in registers; the rows of the survivors are then OR-ed
// into the removed bit vector by all threads at once -- (survivor, word) items are independent loads, merged with
// shared-memory atomicOr (commutative: the result does not depend on the order).
__global__ void __launch_bounds__(kScanThreads) nms_scan_kernel(const __grid_constant__ NmsParams p) {
    DD3D_PDL_PROLOGUE();
    const int c = blockIdx.x, b = blockIdx.y;
    const int cap = p.num_levels * p.topk, C = p.num_classes;
    const NmsScratch sc = bind_nms_scratch(p.scratch, p.B, cap, C);
    const int nc = sc.seg_cnt[b * C + c];
    if (nc <= 1) return;
    const int nblk = (nc + 63) >> 6;
    const size_t row0 = static_cast<size_t>(b) * sc.capP + static_cast<size_t>(sc.seg_blk[b * (C + 1) + c]) * 64;
    const unsigned long long* mask = sc.mask + row0 * sc.W;
    __shared__ unsigned long long s_removed[kScanThreads];
    __shared__ unsigned long long s_diag[2][64];
    __shared__ unsigned long long s_kept;
    const int tid = threadIdx.x;
    s_removed[tid] = 0ull;
    if (tid < 64) s_diag[0][tid] = tid < nc ? mask[static_cast<size_t>(tid) * sc.W] : 0ull;
    __syncthreads();
    for (int blk = 0; blk < nblk; ++blk) {
        const int cn = min(64, nc - blk * 64);
        if (tid == 0) {
            // greedy pass over the 64 x 64 diagonal block: jump from survivor to survivor (one step per KEPT box, not per
            // box): the lowest box still alive is kept and clears everything its diagonal word suppresses
            const unsigned long long* dg = s_diag[blk & 1];
            unsigned long long alive = ~s_removed[blk];
            if (cn < 64) alive &= (1ull << cn) - 1ull;
            unsigned long long kept = 0ull;
            while (alive) {
                const int i = __ffsll(static_cast<long long>(alive)) - 1;
                kept |= 1ull << i;
                alive &= ~(dg[i] | (1ull << i));  // dg[i] holds bits j > i only
            }
            s_removed[blk] = ~kept;  // bits >= cn are never read
            s_kept = kept;
        }
        __syncthreads();
        const int nrem = nblk - blk - 1;  // words after this block
        if (nrem > 0) {
            // next block's diagonal words (static data) ride along with the row loads
            if (tid < 64) {
                const int r = (blk + 1) * 64 + tid;
                s_diag[(blk + 1) & 1][tid] = r < nc ? mask[static_cast<size_t>(r) * sc.W + blk + 1] : 0ull;
            }
            // (row, word) items of the whole 64-row block; rows that were suppressed are skipped by their bit
            const unsigned long long kept = s_kept;
            const unsigned long long* rows = mask + static_cast<size_t>(blk) * 64 * sc.W + blk + 1;
            for (int it = tid; it < 64 * nrem; it += kScanThreads) {
                const int i = it / nrem, w = it - i * nrem;
                if ((kept >> i) & 1ull) {
                    const unsigned long long v = rows[static_cast<size_t>(i) * sc.W + w];
                    if (v) atomicOr(&s_removed[blk + 1 + w], v);
                }
            }
        }
        __syncthreads();
    }
    uint8_t* removed = sc.removed + static_cast<size_t>(b) * cap;
    const uint16_t* cpos = sc.cpos + row0;
    for (int k = tid; k < nc; k += kScanThreads)
        if ((s_removed[k >> 6] >> (k & 63)) & 1ull) removed[cpos[k]] = 1;
}

__global__ void __launch_bounds__(kNmsThreads, 1) nms_finish_kernel(const __grid_constant__ NmsParams p) {
    DD3D_PDL_PROLOGUE();
    extern __shared__ uint8_t smem_raw[];
    const int b = blockIdx.x;
    const int cap = p.num_levels * p.topk;
    NmsSmem m = carve(smem_raw, cap);
    __shared__ int s_warp_sums[33];
    __shared__ int s_base;
    const NmsScratch sc = bind_nms_scratch(p.scratch, p.B, cap, p.num_classes);
    const Det* cand = p.cand + static_cast<size_t>(b) * cap;
    const int n = sc.n[b];
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int slot = sc.order[static_cast<size_t>(b) * cap + i];
        m.val[i] = static_cast<uint16_t>(slot);
        const Det& d = cand[slot];
        m.boxes[i] = make_float4(d.box[0], d.box[1], d.box[2], d.box[3]);
        m.flag[i] = sc.removed[static_cast<size_t>(b) * cap + i] ? 0 : 1;  // keep flags
    }
    __syncthreads();
    finish_image(p, b, cand, m, n, true, s_warp_sums, &s_base);
}

}  // namespace

static int g_class_parallel = -1;
void nms_set_class_parallel(int mode) { g_class_parallel = (mode == 0 || mode == 1) ? mode : -1; }

int nms_class_parallel(const NmsParams& p) {
    if (g_class_parallel < 0) {  // DD3D_NMS_CLASS_PARALLEL=0 / dd3d_set_conv_policy("nms_class_parallel", 0): single-CTA kernel
        const char* e = getenv("DD3D_NMS_CLASS_PARALLEL");
        g_class_parallel = (e && atoi(e) == 0) ? 0 : 1;
    }
    return g_class_parallel && p.scratch != nullptr && p.do_nms && p.nms_thresh > 0.f && p.num_classes >= 1 &&
           p.num_classes <= 255;
}

int nms_launches(const NmsParams& p) { return p.class_parallel ? 4 : 1; }

size_t nms_scratch_bytes(int B, int topk, int num_classes, int num_levels) {
    const int cap = num_levels * topk;
    const NmsScratch sc = bind_nms_scratch(nullptr, B, cap, num_classes);
    return static_cast<size_t>(reinterpret_cast<uintptr_t>(sc.mask)) /* offset: bound at address 0 */ +
           up256(static_cast<size_t>(B) * sc.capP * sc.W * 8);
}

cudaError_t launch_nms(const NmsParams& p, cudaStream_t stream) {
    const int cap = p.num_levels * p.topk;
    if (p.topk > kMaxPreNmsTopk || p.B <= 0 || p.num_levels < 1 || p.num_levels > kLevels) return cudaErrorInvalidValue;
    const size_t smem = nms_smem_bytes(cap);  // key 8 + val 2 per sort entry; box 16 + list 4 + list2 4 + cls 1 + flag 1
    const size_t smem_sort = static_cast<size_t>(cap) * (8 + 2 + 1) + 16;
    static size_t attr_smem_dev[64] = {};  // per device; the limit is 227 KiB minus the static shared memory: ask for what we use
    size_t& attr_smem = attr_smem_dev[current_device_or_zero()];
    if (smem > attr_smem) {
        cudaError_t e = cudaFuncSetAttribute(nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
        if (e == cudaSuccess)
            e = cudaFuncSetAttribute(nms_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxCand * 11 + 16);
        if (e == cudaSuccess)
            e = cudaFuncSetAttribute(nms_finish_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
        if (e != cudaSuccess) {
            cudaGetLastError();
            return e;
        }
        attr_smem = smem;
    }
    if (p.class_parallel) {
        cudaError_t e = launch_pdl(nms_sort_kernel, dim3(kSortCtasPerImage, p.B), dim3(kSortThreads), smem_sort, stream, p);
        if (e == cudaSuccess) e = launch_pdl(nms_mask_kernel, dim3(kMaskCtasPerImage, p.B), dim3(kMaskThreads), 0, stream, p);
        if (e == cudaSuccess) e = launch_pdl(nms_scan_kernel, dim3(p.num_classes, p.B), dim3(kScanThreads), 0, stream, p);
        if (e == cudaSuccess) e = launch_pdl(nms_finish_kernel, dim3(p.B), dim3(kNmsThreads), smem, stream, p);
        return e;
    }
    return launch_pdl(nms_kernel, dim3(p.B), dim3(kNmsThreads), smem, stream, p);
}

}  // namespace dd3d
