// Test-time augmentation on large merged sets: the view merge and the two class-aware greedy NMS forms of the TTA wrappers
// for up to kTtaMaxViews * kLevels * kMaxPreNmsTopk = 92 000 merged detections per image, with scratch linear in the
// number of boxes.
//
//   tta merge   the per-detection inverse transform of tta.cu on the whole GPU (one thread per view slot, view offsets
//               from the prefix of the counts), then detectron2 batched_nms on scores_3d with the axis-aligned IoU
//               (test_time_augmentation.py:164-170); output in descending (scores_3d, Det::index, concatenation index)
//               order, or the plain view-order concatenation without NMS, or (sort-only mode) the concatenation sorted by
//               scores_3d with ties in concatenation order -- the order in which a following order-preserving BEV NMS
//               returns bev_nms's keep (test_time_augmentation.py:172-181);
//   group BEV   the rotated-IoU NMS of bev_geom.cuh per (group of images, class), camera or global frame, the max_dets cap
//               on the survivors of the call and the order-preserving compaction of dd3d_op_group_bev_nms
//               (bev_nms / nuscenes_sample_aggregate, nuscenes_dd3d_tta.py:95-101); ties by image, then slot.
//
// Both NMS forms share one pipeline:
//   sort     stable LSD radix sort (8-bit digits; per pass: tile histograms, one-CTA scan, stable scatter ranked with
//            __match_any_sync), so equal keys keep their input order and the result does not depend on CTA scheduling;
//   bounds   first / last sorted position of every (group, class) segment, geometry gathered in sorted order;
//   nms      one CTA per segment, blocks of kTlBlock sorted rows in order.  Per block: every row is tested against the
//            survivors of the earlier blocks (staged kTlStage at a time in shared memory, first hit wins), then the greedy
//            pass runs inside the block 64 rows at a time (64 x 64 diagonal resolved by one warp, survivors pushed to the
//            later rows of the block), then the block's survivors are appended to the segment's survivor list.  A row is
//            kept iff no earlier kept row of its segment suppresses it: the exact greedy result, ties across block
//            boundaries included, with no N^2 bit matrix: scratch is O(boxes) plus a per-segment bounds table.
// No host synchronisation: every grid is sized from the capacity, and rows past the device-side counts are skipped.
#include <algorithm>

#include "bev_geom.cuh"
#include "device_once.cuh"
#include "pdl.cuh"
#include "tta_view.cuh"

namespace dd3d {

namespace {

constexpr int kTlBlock = 2048;    // sorted rows per block of a segment
constexpr int kTlStage = 1024;    // earlier survivors staged in shared memory per pass
constexpr int kTlThreads = 1024;  // one NMS CTA per segment
constexpr int kTlMergeThreads = 256;
constexpr int kTlPrepThreads = 128;
constexpr int kTlCompactThreads = 1024;
constexpr int kTlMaxB = 256;
constexpr int kTlGroupImages = 16;
constexpr int kTlMaxCls = 128;          // class ids of the grouped BEV NMS (DD3D_MAX_NUM_CLASSES)
constexpr int kTlMergeSegs = 256;       // class segments of the merge NMS: cls & 255, the old kernel's uint8 class compare
constexpr int kTlMergeFlag = 16;        // a view count above cap (same bit as the one-CTA merge's overflow)
constexpr int kTlGroupFlag = 32;        // the grouped BEV NMS's capacity bit
constexpr int kRsThreads = 1024, kRsRounds = 4, kRsTile = kRsThreads * kRsRounds, kRsDigits = 256;

size_t al256(size_t x) { return (x + 255) / 256 * 256; }

// ---------------------------------------------------------------------------------------------- stable radix sort
struct RsParams {
    const uint64_t* kin;
    const int32_t* vin;
    uint64_t* kout;
    int32_t* vout;
    uint32_t* hist;  // [kRsDigits][tiles]
    int n, tiles, shift;
};

__global__ void __launch_bounds__(kRsThreads) rs_hist_kernel(const RsParams p) {
    DD3D_PDL_PROLOGUE();
    __shared__ uint32_t s_h[kRsDigits];
    for (int d = threadIdx.x; d < kRsDigits; d += blockDim.x) s_h[d] = 0u;
    __syncthreads();
    const int t0 = blockIdx.x * kRsTile;
    for (int r = 0; r < kRsRounds; ++r) {
        const int i = t0 + r * kRsThreads + threadIdx.x;
        if (i < p.n) atomicAdd(&s_h[(p.kin[i] >> p.shift) & 255ull], 1u);  // a count: order-independent
    }
    __syncthreads();
    for (int d = threadIdx.x; d < kRsDigits; d += blockDim.x) p.hist[static_cast<size_t>(d) * p.tiles + blockIdx.x] = s_h[d];
}

// exclusive scan of the digit-major histogram in place: each thread a contiguous run, one block scan of the run sums
__global__ void __launch_bounds__(kRsThreads) rs_scan_kernel(const RsParams p) {
    DD3D_PDL_PROLOGUE();
    __shared__ uint32_t s_sum[kRsThreads];
    const size_t M = static_cast<size_t>(kRsDigits) * p.tiles;
    const size_t per = (M + kRsThreads - 1) / kRsThreads;
    const size_t b = threadIdx.x * per, e = b + per < M ? b + per : M;
    uint32_t s = 0u;
    for (size_t i = b; i < e; ++i) s += p.hist[i];
    s_sum[threadIdx.x] = s;
    __syncthreads();
    for (int o = 1; o < kRsThreads; o <<= 1) {
        const uint32_t v = threadIdx.x >= o ? s_sum[threadIdx.x - o] : 0u;
        __syncthreads();
        s_sum[threadIdx.x] += v;
        __syncthreads();
    }
    uint32_t run = threadIdx.x ? s_sum[threadIdx.x - 1] : 0u;
    for (size_t i = b; i < e; ++i) {
        const uint32_t v = p.hist[i];
        p.hist[i] = run;
        run += v;
    }
}

// Stable scatter of one tile: elements in index order (round, warp, lane); rank among equal digits = earlier warps of the
// round (per-warp digit counts, scanned per digit) + earlier lanes of the warp (__match_any_sync peers).
__global__ void __launch_bounds__(kRsThreads) rs_scatter_kernel(const RsParams p) {
    DD3D_PDL_PROLOGUE();
    __shared__ uint32_t s_w[kRsThreads / 32][kRsDigits];
    __shared__ uint32_t s_base[kRsDigits];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int d = threadIdx.x; d < kRsDigits; d += blockDim.x) s_base[d] = p.hist[static_cast<size_t>(d) * p.tiles + blockIdx.x];
    const int t0 = blockIdx.x * kRsTile;
    for (int r = 0; r < kRsRounds; ++r) {
        for (int k = threadIdx.x; k < (kRsThreads / 32) * kRsDigits; k += blockDim.x) (&s_w[0][0])[k] = 0u;
        __syncthreads();
        const int i = t0 + r * kRsThreads + threadIdx.x;
        const bool valid = i < p.n;
        const uint64_t key = valid ? p.kin[i] : 0ull;
        const int32_t val = valid ? p.vin[i] : 0;
        const int d = valid ? static_cast<int>((key >> p.shift) & 255ull) : kRsDigits;
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        const int rank = __popc(peers & ((1u << lane) - 1u));
        if (valid && rank == 0) s_w[warp][d] = __popc(peers);
        __syncthreads();
        if (threadIdx.x < kRsDigits) {
            uint32_t run = s_base[threadIdx.x];
            for (int w = 0; w < kRsThreads / 32; ++w) {
                const uint32_t c = s_w[w][threadIdx.x];
                s_w[w][threadIdx.x] = run;
                run += c;
            }
            s_base[threadIdx.x] = run;
        }
        __syncthreads();
        if (valid) {
            const uint32_t pos = s_w[warp][d] + rank;
            p.kout[pos] = key;
            p.vout[pos] = val;
        }
        __syncthreads();  // s_w is cleared by the next round
    }
}

size_t rs_hist_words(int n) { return static_cast<size_t>(kRsDigits) * ((n + kRsTile - 1) / kRsTile); }

// Stable sort of n (key, value) pairs on key bits [begin, end): ping-pongs between (k[0], v[0]) and (k[1], v[1]); the
// result lands in buffer *which.
cudaError_t radix_sort(uint64_t* const k[2], int32_t* const v[2], uint32_t* hist, int n, int begin, int end, int* which,
                       cudaStream_t stream) {
    RsParams p{};
    p.hist = hist;
    p.n = n;
    p.tiles = (n + kRsTile - 1) / kRsTile;
    int cur = 0;
    cudaError_t e = cudaSuccess;
    for (int shift = begin; shift < end && e == cudaSuccess; shift += 8, cur ^= 1) {
        p.kin = k[cur];
        p.vin = v[cur];
        p.kout = k[cur ^ 1];
        p.vout = v[cur ^ 1];
        p.shift = shift;
        e = launch_pdl(rs_hist_kernel, dim3(p.tiles), dim3(kRsThreads), 0, stream, p);
        if (e == cudaSuccess) e = launch_pdl(rs_scan_kernel, dim3(1), dim3(kRsThreads), 0, stream, p);
        if (e == cudaSuccess) e = launch_pdl(rs_scatter_kernel, dim3(p.tiles), dim3(kRsThreads), 0, stream, p);
    }
    *which = cur;
    return e;
}

int bit_length(unsigned x) {
    int b = 0;
    while (x) {
        ++b;
        x >>= 1;
    }
    return b;
}

// ---------------------------------------------------------------------------------------------- blocked greedy NMS
struct TlBox {  // axis-aligned 2-D box (x1, y1, x2, y2)
    float4 b;
};
struct TlRect {  // BEV rectangle (cx, cy, w, h, angle in degrees)
    float r[5];
};

// `a` precedes `c` in the score order: the argument order of the existing kernels (the rotated clipper is not symmetric)
__device__ __forceinline__ bool tl_hit(const TlBox& a, const TlBox& c, float thr) { return iou_tv(a.b, c.b) > thr; }
__device__ __forceinline__ bool tl_hit(const TlRect& a, const TlRect& c, float thr) {
    return !(thr >= 0.f && circles_apart(a.r, c.r)) && rotated_iou(a.r, c.r) > thr;
}

template <class G>
struct TlNms {
    const G* geom;           // [N] by sorted position
    const int32_t* seg_lo;   // [segments] first sorted position of the segment (lo == hi: empty)
    const int32_t* seg_hi;   // [segments] one past its last
    const int32_t* keep_at;  // [N] index of keep[] that receives the decision of sorted position i
    G* surv;                 // [N] survivors of a segment, packed from the segment's first position
    uint8_t* keep;
    float thr;
    int suppress;            // 0: every row is kept
};

template <class G>
constexpr size_t tl_nms_smem() {
    return static_cast<size_t>(kTlBlock + kTlStage) * sizeof(G) + kTlBlock;
}

template <class G>
__global__ void __launch_bounds__(kTlThreads) tl_nms_kernel(const TlNms<G> p) {
    DD3D_PDL_PROLOGUE();
    extern __shared__ __align__(16) unsigned char tl_smem[];
    G* s_blk = reinterpret_cast<G*>(tl_smem);
    G* s_stage = s_blk + kTlBlock;
    uint8_t* s_dead = reinterpret_cast<uint8_t*>(s_stage + kTlStage);
    __shared__ unsigned long long s_diag[64];
    __shared__ unsigned long long s_kept;
    __shared__ int s_warp[kTlThreads / 32];
    const int start = p.seg_lo[blockIdx.x], n = p.seg_hi[blockIdx.x] - start;
    if (n <= 0) return;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int nsurv = 0;  // block-uniform
    for (int b0 = 0; b0 < n; b0 += kTlBlock) {
        const int R = min(kTlBlock, n - b0);
        for (int i = tid; i < R; i += blockDim.x) {
            s_blk[i] = p.geom[start + b0 + i];
            s_dead[i] = 0;
        }
        __syncthreads();
        if (p.suppress) {
            // 1. the survivors of the earlier blocks, kTlStage at a time
            for (int k0 = 0; k0 < nsurv; k0 += kTlStage) {
                const int ks = min(kTlStage, nsurv - k0);
                for (int k = tid; k < ks; k += blockDim.x) s_stage[k] = p.surv[start + k0 + k];
                __syncthreads();
                for (int i = tid; i < R; i += blockDim.x) {
                    if (s_dead[i]) continue;
                    const G a = s_blk[i];
                    for (int k = 0; k < ks; ++k)
                        if (tl_hit(s_stage[k], a, p.thr)) {
                            s_dead[i] = 1;
                            break;
                        }
                }
                __syncthreads();
            }
            // 2. greedy inside the block, 64 rows at a time: 16 threads per row of the 64 x 64 diagonal
            for (int c0 = 0; c0 < R; c0 += 64) {
                const int cn = min(64, R - c0);
                {
                    const int i = tid >> 4, part = tid & 15;
                    unsigned long long m = 0ull;
                    if (i < cn && !s_dead[c0 + i]) {
                        const G a = s_blk[c0 + i];
#pragma unroll
                        for (int u = 0; u < 4; ++u) {
                            const int j = part * 4 + u;
                            if (j > i && j < cn && !s_dead[c0 + j] && tl_hit(a, s_blk[c0 + j], p.thr)) m |= 1ull << j;
                        }
                    }
#pragma unroll
                    for (int o = 1; o < 16; o <<= 1) m |= __shfl_xor_sync(0xffffffffu, m, o);
                    if (part == 0) s_diag[i] = m;
                }
                __syncthreads();
                if (tid < 32) {
                    const unsigned r_lo = __ballot_sync(0xffffffffu, lane < cn && s_dead[c0 + lane]);
                    const unsigned r_hi = __ballot_sync(0xffffffffu, lane + 32 < cn && s_dead[c0 + lane + 32]);
                    unsigned long long removed = (static_cast<unsigned long long>(r_hi) << 32) | r_lo;
                    if (cn < 64) removed |= ~0ull << cn;
                    unsigned long long kept = 0ull;
                    for (int i = 0; i < 64; ++i)
                        if (!((removed >> i) & 1ull)) {
                            kept |= 1ull << i;
                            removed |= s_diag[i];
                        }
                    if (lane == 0) s_kept = kept;
                    if (lane < cn) s_dead[c0 + lane] = ((kept >> lane) & 1ull) ? 0 : 1;
                    if (lane + 32 < cn) s_dead[c0 + lane + 32] = ((kept >> (lane + 32)) & 1ull) ? 0 : 1;
                }
                __syncthreads();
                const unsigned long long kept = s_kept;
                if (kept)
                    for (int k = c0 + cn + tid; k < R; k += blockDim.x) {
                        if (s_dead[k]) continue;
                        const G c = s_blk[k];
                        for (unsigned long long m = kept; m; m &= m - 1)
                            if (tl_hit(s_blk[c0 + __ffsll(static_cast<long long>(m)) - 1], c, p.thr)) {
                                s_dead[k] = 1;
                                break;
                            }
                    }
                __syncthreads();
            }
        }
        // 3. decisions of the block; its survivors join the segment's list in sorted order
        for (int s0 = 0; s0 < R; s0 += blockDim.x) {
            const int i = s0 + tid;
            const bool alive = i < R && !s_dead[i];
            const unsigned ballot = __ballot_sync(0xffffffffu, alive);
            if (lane == 0) s_warp[warp] = __popc(ballot);
            __syncthreads();
            int off = nsurv, total = nsurv;
            for (int w = 0; w < kTlThreads / 32; ++w) {
                if (w < warp) off += s_warp[w];
                total += s_warp[w];
            }
            if (i < R) {
                p.keep[p.keep_at[start + b0 + i]] = alive ? 1 : 0;
                if (alive && p.suppress) p.surv[start + off + __popc(ballot & ((1u << lane) - 1u))] = s_blk[i];
            }
            nsurv = total;
            __syncthreads();  // s_warp is rewritten by the next chunk
        }
    }
}

template <class G>
cudaError_t launch_tl_nms(const TlNms<G>& p, int segments, cudaStream_t stream) {
    static uint64_t configured_devices = 0;
    if (first_use_on_device(&configured_devices)) {
        const cudaError_t e = cudaFuncSetAttribute(tl_nms_kernel<G>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                   static_cast<int>(tl_nms_smem<G>()));
        if (e != cudaSuccess) return e;
    }
    return launch_pdl(tl_nms_kernel<G>, dim3(segments), dim3(kTlThreads), tl_nms_smem<G>(), stream, p);
}

// ---------------------------------------------------------------------------------------------- TTA merge
struct TmParams {
    const Det* dets;        // [A][cap]
    const int32_t* counts;  // [A]
    TtaView view[kTtaMaxViews];
    Det* cand;              // [A * cap] concatenation (do_nms)
    Det* out;               // [A * cap]
    int32_t* out_count;
    int32_t* total;         // [1] merged detections
    int32_t* flags;
    uint64_t* key;          // [N] pass-1 keys: ~scores_3d bits << 32 | Det::index; padding ~0
    int32_t* val;           // [N] concatenation index
    const uint64_t* key1;   // pass-1 result
    const int32_t* val1;
    uint64_t* key2;         // [N] pass-2 keys: cls & 255, padding kTlMergeSegs
    int32_t* val2;          // [N] pass-1 position
    const uint64_t* key2s;  // pass-2 result
    const int32_t* val2s;
    TlBox* geom;
    int32_t* seg_lo;
    int32_t* seg_hi;
    const uint8_t* keep;    // by pass-1 position
    int A, cap, N;
    int do_nms;             // 0: concatenation; 1: sort + NMS; 2: sort by scores_3d only (ties in concatenation order)
    int suppress;
};

__device__ __forceinline__ int tm_offsets(const TmParams& p, int* s_off) {
    if (threadIdx.x == 0) {
        int off = 0;
        for (int a = 0; a < p.A; ++a) {
            s_off[a] = off;
            off += min(max(p.counts[a], 0), p.cap);
        }
        s_off[p.A] = off;
    }
    __syncthreads();
    return s_off[p.A];
}

// grid (cap / kTlMergeThreads, A): slot s of view a -> concatenation index off[a] + s (view order, like the one-CTA merge)
__global__ void __launch_bounds__(kTlMergeThreads) tm_merge_kernel(const TmParams p) {
    DD3D_PDL_PROLOGUE();
    __shared__ int s_off[kTtaMaxViews + 1];
    __shared__ float s_iK[9];
    const int a = blockIdx.y;
    if (threadIdx.x == 0) tta_inv3(p.view[a].K_view, s_iK);
    const int total = tm_offsets(p, s_off);
    if (blockIdx.x == 0 && a == 0) {
        for (int t = threadIdx.x; t < kTlMergeSegs; t += blockDim.x) p.seg_lo[t] = p.seg_hi[t] = 0;
        if (threadIdx.x == 0) {
            *p.total = total;
            if (p.do_nms == 0) *p.out_count = total;
        }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0 && p.counts[a] > p.cap) atomicOr(p.flags, kTlMergeFlag);
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= p.cap) return;
    const int n = s_off[a + 1] - s_off[a];
    if (s >= n) {  // padding of the sort: after every detection, in a fixed order
        if (p.do_nms != 0) {
            const int pad = total + a * p.cap - s_off[a] + (s - n);
            p.key[pad] = ~0ull;
            p.val[pad] = pad;
        }
        return;
    }
    float iK[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) iK[k] = s_iK[k];
    Det d = p.dets[static_cast<size_t>(a) * p.cap + s];
    tta_invert_det(d, p.view[a], iK, a);
    const int c = s_off[a] + s;
    if (p.do_nms != 0) {
        p.cand[c] = d;
        // the one-CTA NMS key with level 0: scores_3d descending, then Det::index; the stable sort adds the concatenation.
        // Sort-only mode: scores_3d alone, ties in concatenation order (the stable argsort of batched_nms_rotated's keep)
        p.key[c] = (static_cast<uint64_t>(~__float_as_uint(d.score3d)) << 32) |
                   (p.do_nms == 1 ? static_cast<uint32_t>(d.index) : 0u);
        p.val[c] = c;
    } else {
        p.out[c] = d;
    }
}

__global__ void __launch_bounds__(kTlMergeThreads) tm_class_key_kernel(const TmParams p) {
    DD3D_PDL_PROLOGUE();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.N) return;
    const int c = p.val1[i];
    p.key2[i] = c < *p.total ? static_cast<uint64_t>(p.cand[c].cls & 255) : static_cast<uint64_t>(kTlMergeSegs);
    p.val2[i] = i;
}

__global__ void __launch_bounds__(kTlMergeThreads) tm_bounds_kernel(const TmParams p) {
    DD3D_PDL_PROLOGUE();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.N) return;
    const uint64_t seg = p.key2s[i];
    if (seg >= static_cast<uint64_t>(kTlMergeSegs)) return;
    if (i == 0 || p.key2s[i - 1] != seg) p.seg_lo[seg] = i;
    if (i == p.N - 1 || p.key2s[i + 1] != seg) p.seg_hi[seg] = i + 1;
    const Det& d = p.cand[p.val1[p.val2s[i]]];
    p.geom[i].b = make_float4(d.box[0], d.box[1], d.box[2], d.box[3]);
}

// survivors in pass-1 order (descending scores_3d): one CTA, order-preserving
__global__ void __launch_bounds__(kTlCompactThreads) tm_compact_kernel(const TmParams p) {
    DD3D_PDL_PROLOGUE();
    __shared__ int s_warp[kTlCompactThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int total = *p.total;
    int base = 0;
    for (int s0 = 0; s0 < total; s0 += blockDim.x) {
        const int j = s0 + threadIdx.x;
        const bool keep = j < total && (p.do_nms == 2 || p.keep[j]);
        const unsigned ballot = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) s_warp[warp] = __popc(ballot);
        __syncthreads();
        int off = base, sum = base;
        for (int w = 0; w < kTlCompactThreads / 32; ++w) {
            if (w < warp) off += s_warp[w];
            sum += s_warp[w];
        }
        if (keep) p.out[off + __popc(ballot & ((1u << lane) - 1u))] = p.cand[p.val1[j]];
        base = sum;
        __syncthreads();
    }
    if (threadIdx.x == 0) *p.out_count = base;
}

struct TmScratch {
    size_t cand, total, key[2], val[2], key2[2], val2[2], hist, geom, surv, keep, seg_lo, seg_hi, bytes;
};

TmScratch tm_layout(int A, int cap) {
    const size_t N = static_cast<size_t>(A) * cap;
    TmScratch s;
    size_t o = 0;
    auto take = [&](size_t bytes) {
        const size_t at = o;
        o += al256(bytes);
        return at;
    };
    s.cand = take(N * sizeof(Det));
    s.total = take(4);
    for (int b = 0; b < 2; ++b) {
        s.key[b] = take(N * 8);
        s.val[b] = take(N * 4);
        s.key2[b] = take(N * 8);
        s.val2[b] = take(N * 4);
    }
    s.hist = take(rs_hist_words(static_cast<int>(N)) * 4);
    s.geom = take(N * sizeof(TlBox));
    s.surv = take(N * sizeof(TlBox));
    s.keep = take(N);
    s.seg_lo = take(kTlMergeSegs * 4);
    s.seg_hi = take(kTlMergeSegs * 4);
    s.bytes = o;
    return s;
}

// ---------------------------------------------------------------------------------------------- grouped BEV NMS
struct GlParams {
    Det* dets;             // [B][cap], compacted in place
    int32_t* counts;       // [B]
    const float* view_K;   // [B][num_views][9]
    const float* poses;    // [B][7], global mode
    const int32_t* group;  // [B]
    float* global;         // [B][cap][10] or nullptr
    int32_t* flags;
    int B, cap, N, num_views, pose_mode, num_groups, max_group_images, max_dets, segments;
    float thr;
    int32_t* img_n;        // [B] boxes of image b that enter the NMS
    uint64_t* key;         // [N] by slot: (group * 128 + class) << 32 | ~scores_3d bits; padding segments << 32
    int32_t* val;          // [N] slot b * cap + s
    const uint64_t* keys;  // sorted
    const int32_t* vals;
    TlRect* rect;          // [N] by slot
    TlRect* geom;          // [N] by sorted position
    int32_t* seg_lo;
    int32_t* seg_hi;
    uint8_t* keep;         // [N] by slot
    unsigned long long* sel;  // [2] key of the max_dets-th survivor, capped
};

__global__ void __launch_bounds__(256) gl_layout_kernel(const GlParams p) {
    DD3D_PDL_PROLOGUE();
    __shared__ int s_imgs[kTlMaxB];
    for (int t = threadIdx.x; t < p.segments; t += blockDim.x) p.seg_lo[t] = p.seg_hi[t] = 0;
    if (threadIdx.x != 0) return;
    for (int g = 0; g < p.num_groups; ++g) s_imgs[g] = 0;
    int bad = 0;
    for (int b = 0; b < p.B; ++b) {  // the images of a group in call order; one past max_group_images is dropped
        const int g = p.group[b];
        p.img_n[b] = 0;
        if (g < 0 || g >= p.num_groups || s_imgs[g] == p.max_group_images) {
            bad = 1;
            continue;
        }
        if (p.counts[b] > p.cap) bad = 1;  // fail loudly rather than truncate
        ++s_imgs[g];
        p.img_n[b] = min(max(p.counts[b], 0), p.cap);
    }
    if (bad) atomicOr(p.flags, kTlGroupFlag);
}

// pose_cam_global = CAMERA_TO_VEHICLE_ROTATION (bev_nms.py:27-32)
__constant__ float kTlCamToVehicle[9] = {0.f, 0.f, 1.f, -1.f, 0.f, 0.f, 0.f, -1.f, 0.f};

__global__ void __launch_bounds__(kTlPrepThreads) gl_prep_kernel(const GlParams p) {
    DD3D_PDL_PROLOGUE();
    const int b = blockIdx.y, s = blockIdx.x * kTlPrepThreads + threadIdx.x;
    if (s >= p.cap) return;
    const int flat = b * p.cap + s;
    p.keep[flat] = 0;
    p.val[flat] = flat;
    if (s >= p.img_n[b]) {
        p.key[flat] = static_cast<uint64_t>(p.segments) << 32;
        return;
    }
    const Det& D = p.dets[flat];
    int view = p.num_views > 1 ? D.level : 0;
    if (view < 0 || view >= p.num_views) {
        atomicOr(p.flags, kTlGroupFlag);
        view = 0;
    }
    float iK[9], Rw[9], R[9], t[3];
    TlRect rc;
    invert_K(p.view_K + (static_cast<size_t>(b) * p.num_views + view) * 9, iK);
    const float zero[3] = {0.f, 0.f, 0.f};
    const float* pose_t = zero;
    if (p.pose_mode == 0) {
        quat_to_mat3(p.poses + b * 7, Rw);
        pose_t = p.poses + b * 7 + 4;
    } else {
#pragma unroll
        for (int i = 0; i < 9; ++i) Rw[i] = kTlCamToVehicle[i];
    }
    box_to_global(D, iK, Rw, pose_t, R, t, rc.r);
    p.rect[flat] = rc;
    if (p.global) {
        float q[4];
        mat3_to_quat(R, q);
        float* go = p.global + static_cast<size_t>(flat) * 10;
        go[0] = q[0]; go[1] = q[1]; go[2] = q[2]; go[3] = q[3];
        go[4] = t[0]; go[5] = t[1]; go[6] = t[2];
        go[7] = D.size[0]; go[8] = D.size[1]; go[9] = D.size[2];
    }
    int cls = D.cls;
    if (cls < 0 || cls >= kTlMaxCls) {
        atomicOr(p.flags, kTlGroupFlag);
        cls = min(max(cls, 0), kTlMaxCls - 1);
    }
    // (group, class) major; descending scores_3d (non-negative floats order like their bit patterns); the stable sort
    // keeps slot order -- image order inside a group, then slot: the concatenation order of the grouped kernels
    p.key[flat] = (static_cast<uint64_t>(p.group[b] * kTlMaxCls + cls) << 32) | ~__float_as_uint(D.score3d);
}

__global__ void __launch_bounds__(kTlMergeThreads) gl_bounds_kernel(const GlParams p) {
    DD3D_PDL_PROLOGUE();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.N) return;
    const uint64_t seg = p.keys[i] >> 32;
    if (seg >= static_cast<uint64_t>(p.segments)) return;
    if (i == 0 || (p.keys[i - 1] >> 32) != seg) p.seg_lo[seg] = i;
    if (i == p.N - 1 || (p.keys[i + 1] >> 32) != seg) p.seg_hi[seg] = i + 1;
    p.geom[i] = p.rect[p.vals[i]];
}

__device__ __forceinline__ float gl_keep_score(const GlParams& p, int flat) {
    return p.keep[flat] ? p.dets[flat].score3d : -1.0f;
}

// key of a survivor in the NMS output order of the whole call: scores_3d descending, then image, then slot
__device__ __forceinline__ unsigned long long gl_survivor_key(float score, int flat) {
    return (static_cast<unsigned long long>(~__float_as_uint(score)) << 32) | static_cast<unsigned long long>(flat);
}

// radix select of the max_dets-th survivor key of the call (keys are unique: "key <= it" keeps exactly max_dets)
__global__ void __launch_bounds__(kTlCompactThreads) gl_select_kernel(const GlParams p) {
    DD3D_PDL_PROLOGUE();
    __shared__ unsigned s_hist[256];
    __shared__ int s_total, s_k;
    __shared__ unsigned long long s_prefix;
    if (threadIdx.x == 0) s_total = 0;
    __syncthreads();
    if (p.max_dets > 0) {
        int part = 0;
        for (int i = threadIdx.x; i < p.N; i += blockDim.x) part += gl_keep_score(p, i) >= 0.f;
        atomicAdd(&s_total, part);
    }
    __syncthreads();
    if (p.max_dets <= 0 || s_total <= p.max_dets) {
        if (threadIdx.x == 0) {
            p.sel[0] = ~0ull;
            p.sel[1] = 0ull;
        }
        return;
    }
    if (threadIdx.x == 0) {
        s_k = p.max_dets;
        s_prefix = 0ull;
    }
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (int d = threadIdx.x; d < 256; d += blockDim.x) s_hist[d] = 0u;
        __syncthreads();
        const unsigned long long prefix = s_prefix;
        const unsigned long long high = shift == 56 ? 0ull : (~0ull << (shift + 8));
        for (int i = threadIdx.x; i < p.N; i += blockDim.x) {
            const float sc = gl_keep_score(p, i);
            if (sc < 0.f) continue;
            const unsigned long long k = gl_survivor_key(sc, i);
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

// One CTA per image, in place: every write of a chunk lands at or before its own slot, after the chunk's reads.
__global__ void __launch_bounds__(kTlCompactThreads) gl_compact_kernel(const GlParams p) {
    DD3D_PDL_PROLOGUE();
    __shared__ int s_warp[kTlCompactThreads / 32];
    const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const bool capped = p.sel[1] != 0ull;
    const unsigned long long last = p.sel[0];
    int base = 0;
    for (int s0 = 0; s0 < p.cap; s0 += blockDim.x) {
        const int s = s0 + threadIdx.x;
        const int flat = b * p.cap + s;
        bool keep = false;
        Det d;
        float gl[10];
        if (s < p.cap) {
            const float sc = gl_keep_score(p, flat);
            keep = sc >= 0.f && (!capped || gl_survivor_key(sc, flat) <= last);
            if (keep) {
                d = p.dets[flat];
                if (p.global)
#pragma unroll
                    for (int e = 0; e < 10; ++e) gl[e] = p.global[static_cast<size_t>(flat) * 10 + e];
            }
        }
        const unsigned ballot = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) s_warp[warp] = __popc(ballot);
        __syncthreads();
        int off = base, total = base;
        for (int w = 0; w < static_cast<int>(blockDim.x) / 32; ++w) {
            if (w < warp) off += s_warp[w];
            total += s_warp[w];
        }
        if (keep) {
            const size_t to = static_cast<size_t>(b) * p.cap + off + __popc(ballot & ((1u << lane) - 1u));
            p.dets[to] = d;
            if (p.global)
#pragma unroll
                for (int e = 0; e < 10; ++e) p.global[to * 10 + e] = gl[e];
        }
        base = total;
        __syncthreads();
    }
    if (threadIdx.x == 0) p.counts[b] = base;
}

struct GlScratch {
    size_t img_n, key[2], val[2], hist, rect, geom, surv, keep, seg_lo, seg_hi, sel, bytes;
};

GlScratch gl_layout(int B, int cap) {
    const size_t N = static_cast<size_t>(B) * cap;
    const size_t segments = static_cast<size_t>(B) * kTlMaxCls;  // num_groups <= B
    GlScratch s;
    size_t o = 0;
    auto take = [&](size_t bytes) {
        const size_t at = o;
        o += al256(bytes);
        return at;
    };
    s.img_n = take(static_cast<size_t>(B) * 4);
    for (int b = 0; b < 2; ++b) {
        s.key[b] = take(N * 8);
        s.val[b] = take(N * 4);
    }
    s.hist = take(rs_hist_words(static_cast<int>(N)) * 4);
    s.rect = take(N * sizeof(TlRect));
    s.geom = take(N * sizeof(TlRect));
    s.surv = take(N * sizeof(TlRect));
    s.keep = take(N);
    s.seg_lo = take(segments * 4);
    s.seg_hi = take(segments * 4);
    s.sel = take(16);
    s.bytes = o;
    return s;
}

}  // namespace

int tta_merged_cap_large(int A, int cap) {
    if (A < 1 || A > kTtaMaxViews || cap < 1 || cap > kLevels * kMaxPreNmsTopk) return -1;
    return A * cap;
}

size_t tta_large_scratch_bytes(int A, int cap) {
    if (tta_merged_cap_large(A, cap) < 0) return 0;
    return tm_layout(A, cap).bytes;
}

cudaError_t launch_tta_merge_large(const Det* dets, const int32_t* counts, const TtaView* h_views, int A, int cap,
                                   float nms_thresh, int do_nms, void* scratch, Det* out, int32_t* out_count,
                                   int32_t* flags, cudaStream_t stream) {
    if (tta_merged_cap_large(A, cap) < 0) return cudaErrorInvalidValue;
    const TmScratch L = tm_layout(A, cap);
    uint8_t* s = static_cast<uint8_t*>(scratch);
    TmParams p{};
    p.dets = dets;
    p.counts = counts;
    for (int a = 0; a < A; ++a) p.view[a] = h_views[a];
    p.cand = reinterpret_cast<Det*>(s + L.cand);
    p.out = out;
    p.out_count = out_count;
    p.total = reinterpret_cast<int32_t*>(s + L.total);
    p.flags = flags;
    uint64_t* k1[2] = {reinterpret_cast<uint64_t*>(s + L.key[0]), reinterpret_cast<uint64_t*>(s + L.key[1])};
    int32_t* v1[2] = {reinterpret_cast<int32_t*>(s + L.val[0]), reinterpret_cast<int32_t*>(s + L.val[1])};
    uint64_t* k2[2] = {reinterpret_cast<uint64_t*>(s + L.key2[0]), reinterpret_cast<uint64_t*>(s + L.key2[1])};
    int32_t* v2[2] = {reinterpret_cast<int32_t*>(s + L.val2[0]), reinterpret_cast<int32_t*>(s + L.val2[1])};
    uint32_t* hist = reinterpret_cast<uint32_t*>(s + L.hist);
    p.key = k1[0];
    p.val = v1[0];
    p.key2 = k2[0];
    p.val2 = v2[0];
    p.geom = reinterpret_cast<TlBox*>(s + L.geom);
    p.seg_lo = reinterpret_cast<int32_t*>(s + L.seg_lo);
    p.seg_hi = reinterpret_cast<int32_t*>(s + L.seg_hi);
    p.keep = s + L.keep;
    p.A = A;
    p.cap = cap;
    p.N = A * cap;
    p.do_nms = do_nms == 2 ? 2 : (do_nms ? 1 : 0);
    p.suppress = p.do_nms == 1 && nms_thresh > 0.f;  // the one-CTA kernel's rule: no suppression at a threshold <= 0
    cudaError_t e = launch_pdl(tm_merge_kernel, dim3((cap + kTlMergeThreads - 1) / kTlMergeThreads, A),
                               dim3(kTlMergeThreads), 0, stream, p);
    if (e != cudaSuccess || !do_nms) return e;
    const int grid = (p.N + kTlMergeThreads - 1) / kTlMergeThreads;
    int w1 = 0, w2 = 0;
    e = radix_sort(k1, v1, hist, p.N, p.do_nms == 2 ? 32 : 0, 64, &w1, stream);
    p.key1 = k1[w1];
    p.val1 = v1[w1];
    if (e == cudaSuccess && p.do_nms == 2)  // sort only: the concatenation in pass-1 order
        return launch_pdl(tm_compact_kernel, dim3(1), dim3(kTlCompactThreads), 0, stream, p);
    if (e == cudaSuccess) e = launch_pdl(tm_class_key_kernel, dim3(grid), dim3(kTlMergeThreads), 0, stream, p);
    if (e == cudaSuccess) e = radix_sort(k2, v2, hist, p.N, 0, bit_length(kTlMergeSegs), &w2, stream);
    p.key2s = k2[w2];
    p.val2s = v2[w2];
    if (e == cudaSuccess) e = launch_pdl(tm_bounds_kernel, dim3(grid), dim3(kTlMergeThreads), 0, stream, p);
    if (e == cudaSuccess) {
        TlNms<TlBox> q{};
        q.geom = p.geom;
        q.seg_lo = p.seg_lo;
        q.seg_hi = p.seg_hi;
        q.keep_at = p.val2s;  // pass-1 position of each class-major row
        q.surv = reinterpret_cast<TlBox*>(s + L.surv);
        q.keep = s + L.keep;
        q.thr = nms_thresh;
        q.suppress = p.suppress;
        e = launch_tl_nms(q, kTlMergeSegs, stream);
    }
    if (e == cudaSuccess) e = launch_pdl(tm_compact_kernel, dim3(1), dim3(kTlCompactThreads), 0, stream, p);
    return e;
}

static_assert(kTlMaxB == kGroupBevNmsLargeMaxB && kTlGroupImages == kGroupBevNmsLargeGroupImages, "detect.cuh limits");

// layout + prep, the radix passes over (segment, score) keys, bounds, NMS, select, compact: what the launcher enqueues
int group_bev_nms_large_launches(int num_groups) {
    const int key_bits = 32 + bit_length(static_cast<unsigned>(num_groups * kTlMaxCls));
    return 2 + 3 * ((key_bits + 7) / 8) + 4;
}

size_t group_bev_nms_large_scratch_bytes(int B, int cap, int max_group_images) {
    if (B < 1 || B > kTlMaxB || cap < 1 || cap > kTtaMaxViews * kLevels * kMaxPreNmsTopk || max_group_images < 1 ||
        max_group_images > kTlGroupImages)
        return 0;
    return gl_layout(B, cap).bytes;
}

cudaError_t launch_group_bev_nms_large(Det* dets, int32_t* counts, const float* view_K, int num_views, const float* poses,
                                       int pose_mode, const int32_t* group, int num_groups, int max_group_images,
                                       float* global, void* scratch, int32_t* flags, int B, int cap, float thr,
                                       int max_dets, cudaStream_t stream) {
    if (group_bev_nms_large_scratch_bytes(B, cap, max_group_images) == 0 || num_groups < 1 || num_groups > B ||
        num_views < 1 || (pose_mode != 0 && pose_mode != 1) || (pose_mode == 0 && poses == nullptr) || group == nullptr)
        return cudaErrorInvalidValue;
    const GlScratch L = gl_layout(B, cap);
    uint8_t* s = static_cast<uint8_t*>(scratch);
    GlParams p{};
    p.dets = dets;
    p.counts = counts;
    p.view_K = view_K;
    p.poses = poses;
    p.group = group;
    p.global = global;
    p.flags = flags;
    p.B = B;
    p.cap = cap;
    p.N = B * cap;
    p.num_views = num_views;
    p.pose_mode = pose_mode;
    p.num_groups = num_groups;
    p.max_group_images = max_group_images;
    p.max_dets = max_dets;
    p.segments = num_groups * kTlMaxCls;
    p.thr = thr;
    p.img_n = reinterpret_cast<int32_t*>(s + L.img_n);
    uint64_t* k[2] = {reinterpret_cast<uint64_t*>(s + L.key[0]), reinterpret_cast<uint64_t*>(s + L.key[1])};
    int32_t* v[2] = {reinterpret_cast<int32_t*>(s + L.val[0]), reinterpret_cast<int32_t*>(s + L.val[1])};
    p.key = k[0];
    p.val = v[0];
    p.rect = reinterpret_cast<TlRect*>(s + L.rect);
    p.geom = reinterpret_cast<TlRect*>(s + L.geom);
    p.seg_lo = reinterpret_cast<int32_t*>(s + L.seg_lo);
    p.seg_hi = reinterpret_cast<int32_t*>(s + L.seg_hi);
    p.keep = s + L.keep;
    p.sel = reinterpret_cast<unsigned long long*>(s + L.sel);
    cudaError_t e = launch_pdl(gl_layout_kernel, dim3(1), dim3(256), 0, stream, p);
    if (e == cudaSuccess)
        e = launch_pdl(gl_prep_kernel, dim3((cap + kTlPrepThreads - 1) / kTlPrepThreads, B), dim3(kTlPrepThreads), 0,
                       stream, p);
    int w = 0;
    if (e == cudaSuccess)
        e = radix_sort(k, v, reinterpret_cast<uint32_t*>(s + L.hist), p.N, 0, 32 + bit_length(p.segments), &w, stream);
    p.keys = k[w];
    p.vals = v[w];
    if (e == cudaSuccess)
        e = launch_pdl(gl_bounds_kernel, dim3((p.N + kTlMergeThreads - 1) / kTlMergeThreads), dim3(kTlMergeThreads), 0,
                       stream, p);
    if (e == cudaSuccess) {
        TlNms<TlRect> q{};
        q.geom = p.geom;
        q.seg_lo = p.seg_lo;
        q.seg_hi = p.seg_hi;
        q.keep_at = p.vals;  // the slot of each sorted row
        q.surv = reinterpret_cast<TlRect*>(s + L.surv);
        q.keep = p.keep;
        q.thr = thr;
        q.suppress = 1;
        e = launch_tl_nms(q, p.segments, stream);
    }
    if (e == cudaSuccess) e = launch_pdl(gl_select_kernel, dim3(1), dim3(kTlCompactThreads), 0, stream, p);
    if (e == cudaSuccess)
        e = launch_pdl(gl_compact_kernel, dim3(B), dim3(std::min(kTlCompactThreads, (cap + 31) / 32 * 32)), 0, stream, p);
    return e;
}

}  // namespace dd3d
