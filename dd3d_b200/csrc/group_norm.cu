// GroupNorm(32, 256) on NHWC 16-bit views with a channel pitch (FCOS heads / FPN with NORM "GN": fcos2d.py:73-91,
// fcos3d.py:82-100 get_norm("GN") = nn.GroupNorm(32, 256); detectron2 FPN with norm "GN").  Group g holds channels
// [8g, 8g + 8): exactly one 16-byte vector per pixel, so warp lane g owns group g and a warp reads one 512-byte pixel.
//
// Two kernels, one launch each for up to kMaxSeg maps (the five FPN levels of a tower layer):
//   group_norm_stats_kernel  one CTA per (segment, image, chunk of kGnChunk pixels): per-lane running (count, mean, M2) with
//                            Chan's update per pixel, then the 8 warps combined in warp order -> scratch (mean, M2) per
//                            (chunk, group).  No E[x^2] - E[x]^2: a V2-99 p2 group holds 768k values around a non-zero mean.
//   group_norm_apply_kernel  same grid; every CTA first combines the chunks of its (segment, image) in a fixed order
//                            (warp w takes chunks w, w + 8, ...; then warps 0..7), then y = x * s_c + b_c with
//                            s_c = gamma_c * rstd_g, b_c = beta_c - mean_g * s_c, + nearest-2x(residual), * 0.5 (FUSE_TYPE avg),
//                            ReLU; one rounding at the store.  In place is allowed (each pixel is read before it is written
//                            by the same thread).  gamma == nullptr: no statistics, s = 1, b = 0 (the avg fuse of a BN FPN).
// The chunking depends on the map shape only, and every sum runs in a fixed order: bit-identical across launches and
// processes; the scratch is fully written by the stats kernel before the apply kernel reads it.
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

__global__ void __launch_bounds__(kGnThreads) group_norm_stats_kernel(const GroupNormParams p) {
    DD3D_PDL_PROLOGUE();
    __shared__ float sh[kGnWarps][32][3];
    int b, chunk;
    const int s = locate(p, blockIdx.x, &b, &chunk);
    const GroupNormSeg& g = p.seg[s];
    const int HW = g.H * g.W;
    const int p0 = chunk * kGnChunk, p1 = min(HW, p0 + kGnChunk);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const __nv_bfloat16* img = g.in + static_cast<size_t>(b) * HW * g.in_pitch + lane * 8;
    float n = 0.f, mean = 0.f, m2 = 0.f;
#pragma unroll 4
    for (int px = p0 + warp; px < p1; px += kGnWarps) {
        float x[8];
        unpack8(*reinterpret_cast<const uint4*>(img + static_cast<size_t>(px) * g.in_pitch), p.fp16, x);
        const float mb = (((x[0] + x[1]) + (x[2] + x[3])) + ((x[4] + x[5]) + (x[6] + x[7]))) * 0.125f;
        float m2b = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) m2b = fmaf(x[j] - mb, x[j] - mb, m2b);
        chan(n, mean, m2, 8.f, mb, m2b);
    }
    sh[warp][lane][0] = n;
    sh[warp][lane][1] = mean;
    sh[warp][lane][2] = m2;
    __syncthreads();
    if (warp == 0) {
        for (int w = 1; w < kGnWarps; ++w) chan(n, mean, m2, sh[w][lane][0], sh[w][lane][1], sh[w][lane][2]);
        float2* out = g.part + (static_cast<size_t>(b) * g.nchunks + chunk) * 32 + lane;
        *out = make_float2(mean, m2);
    }
}

__global__ void __launch_bounds__(kGnThreads) group_norm_apply_kernel(const GroupNormParams p) {
    DD3D_PDL_PROLOGUE();
    __shared__ float sh[kGnWarps][32][3];
    __shared__ float stat[32][2];  // (mean, rstd) per group
    int b, chunk;
    const int s = locate(p, blockIdx.x, &b, &chunk);
    const GroupNormSeg& g = p.seg[s];
    const int HW = g.H * g.W;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float sc[8], bi[8];
    if (p.gamma != nullptr) {
        float n = 0.f, mean = 0.f, m2 = 0.f;
        const float2* part = g.part + static_cast<size_t>(b) * g.nchunks * 32 + lane;
        for (int c = warp; c < g.nchunks; c += kGnWarps) {
            const float2 v = part[static_cast<size_t>(c) * 32];
            chan(n, mean, m2, 8.f * static_cast<float>(min(kGnChunk, HW - c * kGnChunk)), v.x, v.y);
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
        const float mu = stat[lane][0], rstd = stat[lane][1];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            sc[j] = p.gamma[lane * 8 + j] * rstd;
            bi[j] = p.beta[lane * 8 + j] - mu * sc[j];
        }
    } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            sc[j] = 1.f;
            bi[j] = 0.f;
        }
    }
    const int p0 = chunk * kGnChunk, p1 = min(HW, p0 + kGnChunk);
    const __nv_bfloat16* src = g.in + static_cast<size_t>(b) * HW * g.in_pitch + lane * 8;
    __nv_bfloat16* dst = g.out + static_cast<size_t>(b) * HW * g.out_pitch + lane * 8;
    const __nv_bfloat16* res =
        g.res != nullptr ? g.res + static_cast<size_t>(b) * g.res_H * g.res_W * g.res_pitch + lane * 8 : nullptr;
#pragma unroll 4
    for (int px = p0 + warp; px < p1; px += kGnWarps) {
        float x[8];
        unpack8(*reinterpret_cast<const uint4*>(src + static_cast<size_t>(px) * g.in_pitch), p.fp16, x);
#pragma unroll
        for (int j = 0; j < 8; ++j) x[j] = fmaf(x[j], sc[j], bi[j]);
        if (res != nullptr) {
            const int y = px / g.W, xx = px - y * g.W;
            float r[8];
            unpack8(*reinterpret_cast<const uint4*>(res + (static_cast<size_t>(y >> 1) * g.res_W + (xx >> 1)) * g.res_pitch),
                    p.fp16, r);
#pragma unroll
            for (int j = 0; j < 8; ++j) x[j] += r[j];
        }
        if (p.avg) {
#pragma unroll
            for (int j = 0; j < 8; ++j) x[j] *= 0.5f;
        }
        if (p.relu) {
#pragma unroll
            for (int j = 0; j < 8; ++j) x[j] = fmaxf(x[j], 0.f);
        }
        uint4 o;
        o.x = pack2_act(x[0], x[1], p.fp16);
        o.y = pack2_act(x[2], x[3], p.fp16);
        o.z = pack2_act(x[4], x[5], p.fp16);
        o.w = pack2_act(x[6], x[7], p.fp16);
        *reinterpret_cast<uint4*>(dst + static_cast<size_t>(px) * g.out_pitch) = o;
    }
}

bool aligned16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; }

}  // namespace

int group_norm_chunks(int H, int W) { return (H * W + kGnChunk - 1) / kGnChunk; }

size_t group_norm_scratch_bytes(int B, int H, int W) {
    return static_cast<size_t>(B) * group_norm_chunks(H, W) * 32 * sizeof(float2);
}

cudaError_t launch_group_norm(GroupNormParams p, cudaStream_t stream) {
    if (p.nseg < 1 || p.nseg > kMaxSeg || p.B < 1) return cudaErrorInvalidValue;
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
        if (g.in_pitch < kGnChannels || g.out_pitch < kGnChannels || g.in_pitch % 8 || g.out_pitch % 8) return cudaErrorInvalidValue;
        if (!aligned16(g.in) || !aligned16(g.out)) return cudaErrorInvalidValue;
        if (g.res != nullptr) {
            if (g.res_pitch < kGnChannels || g.res_pitch % 8 || !aligned16(g.res)) return cudaErrorInvalidValue;
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
    if (p.gamma != nullptr) {
        const cudaError_t e = launch_pdl(group_norm_stats_kernel, dim3(static_cast<unsigned>(ctas)), dim3(kGnThreads), 0, stream, p);
        if (e != cudaSuccess) return e;
    }
    return launch_pdl(group_norm_apply_kernel, dim3(static_cast<unsigned>(ctas)), dim3(kGnThreads), 0, stream, p);
}

}  // namespace dd3d
