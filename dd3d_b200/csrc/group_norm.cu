// GroupNorm(32, C) on NHWC 16-bit views with a channel pitch, C = 32 * cpg for cpg in {2, 4, 5, 6, 7, 8, 10, 12, 14, 16, 24,
// 32}: the FCOS heads / FPN with NORM "GN" (fcos2d.py:73-91, fcos3d.py:82-100 get_norm("GN") = nn.GroupNorm(32, C) at every
// FE.FPN.OUT_CHANNELS from 64 to 512; detectron2 FPN with norm "GN") and the VoVNet backbone with FE.BACKBONE.NORM "GN"
// (vovnet.py:119,139,159: 64 .. 1024 channels).
// Thread t of a CTA owns the 16-byte vector v = t % (C / 8) of every pixel it visits (channels [8v, 8v + 8)) and visits the
// pixels r, r + R, ... of its chunk, r = t / (C / 8), R = floor(256 / (C / 8)).  For 256 channels (cpg 8) that is lane = group,
// warp = pixel row: one warp reads one 512-byte pixel.  Where C / 8 does not divide 256 (cpg 5, 6, 7, 10, 12, 14: 20 .. 56
// vectors per pixel) the last 256 - R * C / 8 threads (4 .. 32) own no (vector, row) and only take part in the barriers; the
// mapping is still a function of C alone.  With cpg 5, 6, 7, 10, 12 or 14 a vector holds the ends of two (cpg 5: up to
// three) groups; each thread then keeps one (count, mean, M2) per group it touches (a slot), fixed by v.
//
// Two kernels, one launch each for up to kMaxSeg maps of the same channel count (the five FPN levels of a tower layer):
//   group_norm_stats_kernel  one CTA per (segment, image, chunk of kGnChunk pixels): per-thread running (count, mean, M2) per
//                            slot with Chan's update per pixel, then per group the threads' slots combined in (row, vector)
//                            order -> scratch (mean, M2) per (chunk, group).  No E[x^2] - E[x]^2: a V2-99 p2 group holds 768k
//                            values around a non-zero mean.
//   group_norm_apply_kernel  same grid; every CTA first combines the chunks of its (segment, image) in a fixed order
//                            (warp w takes chunks w, w + 8, ...; then warps 0..7), then y = x * s_c + b_c with
//                            s_c = gamma_c * rstd_g, b_c = beta_c - mean_g * s_c, + nearest-2x(residual), * 0.5 (FUSE_TYPE avg),
//                            ReLU; one rounding at the store.  In place is allowed (each pixel is read before it is written
//                            by the same thread).  gamma == nullptr: no statistics, s = 1, b = 0 (the avg fuse of a BN FPN).
// The chunking depends on the map shape only, and every sum runs in a fixed order: bit-identical across launches, processes
// and batch sizes; the scratch is fully written by the stats kernel before the apply kernel reads it.
#include "act16.cuh"
#include "group_norm.cuh"
#include "pdl.cuh"

namespace dd3d {

namespace {

constexpr int kGnThreads = 256;
constexpr int kGnWarps = kGnThreads / 32;

__device__ __forceinline__ void unpack8(const uint4 u, int fp16, float* x) {
    const float2 a = unpack2_act(u.x, fp16), b = unpack2_act(u.y, fp16), c = unpack2_act(u.z, fp16), d = unpack2_act(u.w, fp16);
    x[0] = a.x; x[1] = a.y; x[2] = b.x; x[3] = b.y; x[4] = c.x; x[5] = c.y; x[6] = d.x; x[7] = d.y;
}

// (n, mean, m2) <- (n, mean, m2) combined with (nb, mb, m2b) (Chan et al.)
__device__ __forceinline__ void chan(float& n, float& mean, float& m2, float nb, float mb, float m2b) {
    const float nn = n + nb;
    if (nn == 0.f) return;
    const float d = mb - mean;
    const float f = nb / nn;
    mean = fmaf(d, f, mean);
    m2 = m2 + m2b + d * d * n * f;
    n = nn;
}

// Thread layout of one channel count (see the file comment)
template <int CPG>
struct GnShape {
    static constexpr int C = 32 * CPG;
    static constexpr int kVec = C / 8;                   // 16-byte vectors per pixel
    static constexpr int kRows = kGnThreads / kVec;      // pixels per CTA step
    static constexpr int slots_of(int v) { return (8 * v + 7) / CPG - 8 * v / CPG + 1; }
    static constexpr int max_slots() {
        int m = 1;
        for (int v = 0; v < kVec; ++v) m = slots_of(v) > m ? slots_of(v) : m;
        return m;
    }
    static constexpr int kSlots = max_slots();           // groups one vector can touch: 1 (cpg % 8 == 0) .. 4 (cpg 2)
    static_assert(C % 8 == 0 && kRows >= 1, "GroupNorm channel count");
};

// segment, image and chunk of CTA `cta`
__device__ __forceinline__ int locate(const GroupNormParams& p, int cta, int* b, int* chunk) {
    int s = 0;
#pragma unroll
    for (int i = 1; i < kMaxSeg; ++i)
        if (i < p.nseg && cta >= p.seg[i].cta0) s = i;
    const int r = cta - p.seg[s].cta0;
    *b = r / p.seg[s].nchunks;
    *chunk = r % p.seg[s].nchunks;
    return s;
}

template <int CPG>
__global__ void __launch_bounds__(kGnThreads) group_norm_stats_kernel(const GroupNormParams p) {
    DD3D_PDL_PROLOGUE();
    using S = GnShape<CPG>;
    constexpr int K = S::kSlots;
    __shared__ float sh[S::kRows * S::kVec][K][3];
    int b, chunk;
    const int s = locate(p, blockIdx.x, &b, &chunk);
    const GroupNormSeg& g = p.seg[s];
    const int HW = g.H * g.W;
    const int p0 = chunk * kGnChunk, p1 = min(HW, p0 + kGnChunk);
    const int v = threadIdx.x % S::kVec, r = threadIdx.x / S::kVec;
    const __nv_bfloat16* img = g.in + static_cast<size_t>(b) * HW * g.in_pitch + v * 8;
    float n[K], mean[K], m2[K];
#pragma unroll
    for (int j = 0; j < K; ++j) n[j] = mean[j] = m2[j] = 0.f;
    if (r < S::kRows) {
        if constexpr (K == 1) {
#pragma unroll 4
            for (int px = p0 + r; px < p1; px += S::kRows) {
                float x[8];
                unpack8(*reinterpret_cast<const uint4*>(img + static_cast<size_t>(px) * g.in_pitch), p.fp16, x);
                const float mb = (((x[0] + x[1]) + (x[2] + x[3])) + ((x[4] + x[5]) + (x[6] + x[7]))) * 0.125f;
                float m2b = 0.f;
#pragma unroll
                for (int k = 0; k < 8; ++k) m2b = fmaf(x[k] - mb, x[k] - mb, m2b);
                chan(n[0], mean[0], m2[0], 8.f, mb, m2b);
            }
        } else {
            // channel k of the vector belongs to slot sl[k] = group - first group of the vector; cnt[j] channels per slot
            const int g0 = 8 * v / CPG;
            int sl[8];
            float cnt[K], inv[K];
#pragma unroll
            for (int k = 0; k < 8; ++k) sl[k] = (8 * v + k) / CPG - g0;
            // channels of group g0 + j inside [8v, 8v + 8), in closed form (a per-channel count left a local-memory array in
            // the cpg 14 instantiation)
#pragma unroll
            for (int j = 0; j < K; ++j)
                cnt[j] = static_cast<float>(max(0, min(8 * v + 8, (g0 + j + 1) * CPG) - max(8 * v, (g0 + j) * CPG)));
#pragma unroll
            for (int j = 0; j < K; ++j) inv[j] = cnt[j] > 0.f ? 1.f / cnt[j] : 0.f;
#pragma unroll 1
            for (int px = p0 + r; px < p1; px += S::kRows) {
                float x[8];
                unpack8(*reinterpret_cast<const uint4*>(img + static_cast<size_t>(px) * g.in_pitch), p.fp16, x);
#pragma unroll
                for (int j = 0; j < K; ++j) {
                    if (cnt[j] == 0.f) continue;
                    float sum = 0.f;
#pragma unroll
                    for (int k = 0; k < 8; ++k) sum += sl[k] == j ? x[k] : 0.f;
                    const float mb = sum * inv[j];
                    float m2b = 0.f;
#pragma unroll
                    for (int k = 0; k < 8; ++k)
                        if (sl[k] == j) m2b = fmaf(x[k] - mb, x[k] - mb, m2b);
                    chan(n[j], mean[j], m2[j], cnt[j], mb, m2b);
                }
            }
        }
#pragma unroll
        for (int j = 0; j < K; ++j) {
            sh[threadIdx.x][j][0] = n[j];
            sh[threadIdx.x][j][1] = mean[j];
            sh[threadIdx.x][j][2] = m2[j];
        }
    }
    __syncthreads();
    if (threadIdx.x < 32) {
        // group gi: the slots of the vectors [v0, v1] that hold its channels, rows in order, then vectors in order
        const int gi = threadIdx.x;
        const int v0 = gi * CPG / 8, v1 = (gi * CPG + CPG - 1) / 8;
        const int j0 = gi - 8 * v0 / CPG;
        float an = sh[v0][j0][0], am = sh[v0][j0][1], a2 = sh[v0][j0][2];
        for (int rr = 0; rr < S::kRows; ++rr)
            for (int vv = v0; vv <= v1; ++vv) {
                if (rr == 0 && vv == v0) continue;
                const int t = rr * S::kVec + vv, j = gi - 8 * vv / CPG;
                chan(an, am, a2, sh[t][j][0], sh[t][j][1], sh[t][j][2]);
            }
        float2* out = g.part + (static_cast<size_t>(b) * g.nchunks + chunk) * 32 + gi;
        *out = make_float2(am, a2);
    }
}

template <int CPG>
__global__ void __launch_bounds__(kGnThreads) group_norm_apply_kernel(const GroupNormParams p) {
    DD3D_PDL_PROLOGUE();
    using S = GnShape<CPG>;
    __shared__ float sh[kGnWarps][32][3];
    __shared__ float stat[32][2];  // (mean, rstd) per group
    int b, chunk;
    const int s = locate(p, blockIdx.x, &b, &chunk);
    const GroupNormSeg& g = p.seg[s];
    const int HW = g.H * g.W;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int v = threadIdx.x % S::kVec, r = threadIdx.x / S::kVec;
    float sc[8], bi[8];
    if (p.gamma != nullptr) {
        float n = 0.f, mean = 0.f, m2 = 0.f;
        const float2* part = g.part + static_cast<size_t>(b) * g.nchunks * 32 + lane;
        for (int c = warp; c < g.nchunks; c += kGnWarps) {
            const float2 pv = part[static_cast<size_t>(c) * 32];
            chan(n, mean, m2, static_cast<float>(CPG) * static_cast<float>(min(kGnChunk, HW - c * kGnChunk)), pv.x, pv.y);
        }
        sh[warp][lane][0] = n;
        sh[warp][lane][1] = mean;
        sh[warp][lane][2] = m2;
        __syncthreads();
        if (warp == 0) {
            for (int w = 1; w < kGnWarps; ++w) chan(n, mean, m2, sh[w][lane][0], sh[w][lane][1], sh[w][lane][2]);
            stat[lane][0] = mean;
            stat[lane][1] = 1.0f / sqrtf(m2 / n + 1e-5f);  // biased variance, eps = 1e-5 (nn.GroupNorm)
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int c = v * 8 + k, gi = c / CPG;
            sc[k] = p.gamma[c] * stat[gi][1];
            bi[k] = p.beta[c] - stat[gi][0] * sc[k];
        }
    } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            sc[k] = 1.f;
            bi[k] = 0.f;
        }
    }
    if (r >= S::kRows) return;
    const int p0 = chunk * kGnChunk, p1 = min(HW, p0 + kGnChunk);
    const __nv_bfloat16* src = g.in + static_cast<size_t>(b) * HW * g.in_pitch + v * 8;
    __nv_bfloat16* dst = g.out + static_cast<size_t>(b) * HW * g.out_pitch + v * 8;
    const __nv_bfloat16* res =
        g.res != nullptr ? g.res + static_cast<size_t>(b) * g.res_H * g.res_W * g.res_pitch + v * 8 : nullptr;
#pragma unroll 4
    for (int px = p0 + r; px < p1; px += S::kRows) {
        float x[8];
        unpack8(*reinterpret_cast<const uint4*>(src + static_cast<size_t>(px) * g.in_pitch), p.fp16, x);
#pragma unroll
        for (int k = 0; k < 8; ++k) x[k] = fmaf(x[k], sc[k], bi[k]);
        if (res != nullptr) {
            const int y = px / g.W, xx = px - y * g.W;
            float rv[8];
            unpack8(*reinterpret_cast<const uint4*>(res + (static_cast<size_t>(y >> 1) * g.res_W + (xx >> 1)) * g.res_pitch),
                    p.fp16, rv);
#pragma unroll
            for (int k = 0; k < 8; ++k) x[k] += rv[k];
        }
        if (p.avg) {
#pragma unroll
            for (int k = 0; k < 8; ++k) x[k] *= 0.5f;
        }
        if (p.relu) {
#pragma unroll
            for (int k = 0; k < 8; ++k) x[k] = fmaxf(x[k], 0.f);
        }
        uint4 o;
        o.x = pack2_act(x[0], x[1], p.fp16);
        o.y = pack2_act(x[2], x[3], p.fp16);
        o.z = pack2_act(x[4], x[5], p.fp16);
        o.w = pack2_act(x[6], x[7], p.fp16);
        *reinterpret_cast<uint4*>(dst + static_cast<size_t>(px) * g.out_pitch) = o;
    }
}

template <int CPG>
cudaError_t launch_cpg(const GroupNormParams& p, unsigned ctas, cudaStream_t stream) {
    if (p.gamma != nullptr) {
        const cudaError_t e = launch_pdl(group_norm_stats_kernel<CPG>, dim3(ctas), dim3(kGnThreads), 0, stream, p);
        if (e != cudaSuccess) return e;
    }
    return launch_pdl(group_norm_apply_kernel<CPG>, dim3(ctas), dim3(kGnThreads), 0, stream, p);
}

bool aligned16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; }

}  // namespace

bool group_norm_channels_ok(int C) {
    switch (C) {
        case 64: case 128: case 160: case 192: case 224: case 256: case 320: case 384: case 448: case 512: case 768: case 1024:
            return true;
        default: return false;
    }
}

int group_norm_chunks(int H, int W) { return (H * W + kGnChunk - 1) / kGnChunk; }

size_t group_norm_scratch_bytes(int B, int H, int W) {
    return static_cast<size_t>(B) * group_norm_chunks(H, W) * 32 * sizeof(float2);
}

cudaError_t launch_group_norm(GroupNormParams p, cudaStream_t stream) {
    if (p.nseg < 1 || p.nseg > kMaxSeg || p.B < 1 || !group_norm_channels_ok(p.C)) return cudaErrorInvalidValue;
    if ((p.gamma == nullptr) != (p.beta == nullptr)) return cudaErrorInvalidValue;
    if (p.gamma == nullptr && p.avg == 0 && p.relu == 0) {
        bool any_res = false;
        for (int s = 0; s < p.nseg; ++s) any_res |= p.seg[s].res != nullptr;
        if (!any_res) return cudaErrorInvalidValue;  // nothing to do: refused rather than a silent copy
    }
    long ctas = 0;
    for (int s = 0; s < p.nseg; ++s) {
        GroupNormSeg& g = p.seg[s];
        if (g.H < 1 || g.W < 1 || !g.in || !g.out) return cudaErrorInvalidValue;
        if (g.in_pitch < p.C || g.out_pitch < p.C || g.in_pitch % 8 || g.out_pitch % 8) return cudaErrorInvalidValue;
        if (!aligned16(g.in) || !aligned16(g.out)) return cudaErrorInvalidValue;
        if (g.res != nullptr) {
            if (g.res_pitch < p.C || g.res_pitch % 8 || !aligned16(g.res)) return cudaErrorInvalidValue;
            if (g.res_H != (g.H + 1) / 2 && g.res_H != g.H / 2) return cudaErrorInvalidValue;
            if (g.res_W != (g.W + 1) / 2 && g.res_W != g.W / 2) return cudaErrorInvalidValue;
            if (g.res_H * 2 < g.H || g.res_W * 2 < g.W) return cudaErrorInvalidValue;  // every output pixel has a source
        }
        if (p.gamma != nullptr && (g.part == nullptr || !aligned16(g.part))) return cudaErrorInvalidValue;
        if (static_cast<long>(g.H) * g.W > 0x7fffffffL / 8) return cudaErrorInvalidValue;
        g.nchunks = group_norm_chunks(g.H, g.W);
        g.cta0 = static_cast<int>(ctas);
        ctas += static_cast<long>(p.B) * g.nchunks;
    }
    if (ctas > 0x7fffffffL) return cudaErrorInvalidValue;
    const unsigned n = static_cast<unsigned>(ctas);
    switch (p.C / 32) {
        case 2: return launch_cpg<2>(p, n, stream);
        case 4: return launch_cpg<4>(p, n, stream);
        case 5: return launch_cpg<5>(p, n, stream);
        case 6: return launch_cpg<6>(p, n, stream);
        case 7: return launch_cpg<7>(p, n, stream);
        case 8: return launch_cpg<8>(p, n, stream);
        case 10: return launch_cpg<10>(p, n, stream);
        case 12: return launch_cpg<12>(p, n, stream);
        case 14: return launch_cpg<14>(p, n, stream);
        case 16: return launch_cpg<16>(p, n, stream);
        case 24: return launch_cpg<24>(p, n, stream);
        default: return launch_cpg<32>(p, n, stream);
    }
}

int group_norm_launches(const GroupNormParams& p) { return p.gamma != nullptr ? 2 : 1; }

}  // namespace dd3d
