// Bandwidth-bound kernels of the DD3D backbone (NHWC bf16, 128-bit vector accesses):
//   preprocess   : (x - mean) / std, zero pad, NCHW -> NHWC(4)        reference core.py:61-72, image_list.py:93-158
//   max-pool     : 2x2/s2 (DLA Tree.downsample, dla.py:224-225), 3x3/s2 ceil (VoVNet, vovnet.py:248-249)
//   eSE          : global avg-pool -> fc -> hsigmoid -> channel scale (+identity)   vovnet.py:169-185,233-236
//   relu         : p7 input (detectron2 LastLevelP6P7)
#include "pdl.cuh"
#include "small_kernels.cuh"

#include "act16.cuh"

#include <cuda_bf16.h>
#include <math.h>

namespace dd3d {

namespace {

// ------------------------------------------------------------------------------------------ preprocess
// One thread = 4 consecutive pixels of a row: three 4-byte (uint8 planes) or 16-byte (fp32 planes) loads and one 32-byte
// store.  (One pixel per thread -- 3 single-byte loads, one 8-byte store -- ran at 20 % of the HBM roof, BENCH_r01.)
template <typename T>
__global__ void __launch_bounds__(256) preprocess_kernel(const T* __restrict__ src, const int* __restrict__ sizes,
                                                         __nv_bfloat16* __restrict__ dst, int B, int Hs, int Ws, int Hp, int Wp,
                                                         int size_stride, float m0, float m1, float m2, float s0, float s1,
                                                         float s2, int fp16, int vec_ok) {
    DD3D_PDL_PROLOGUE();
    const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    const int y = blockIdx.y;
    const int b = blockIdx.z;
    if (x0 >= Wp) return;
    const int h = sizes[size_stride * b], w = sizes[size_stride * b + 1];
    float v[3][4];
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int j = 0; j < 4; ++j) v[c][j] = 0.f;
    const float mean[3] = {m0, m1, m2}, stdv[3] = {s0, s1, s2};
    if (y < h && x0 < w) {
        const size_t plane = static_cast<size_t>(Hs) * Ws;
        const T* p = src + static_cast<size_t>(b) * 3 * plane + static_cast<size_t>(y) * Ws + x0;
        if (vec_ok && x0 + 3 < w) {  // Ws % 4 == 0 and an aligned base: one vector load per plane
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                if (sizeof(T) == 1) {
                    const uchar4 q = __ldg(reinterpret_cast<const uchar4*>(p + c * plane));
                    v[c][0] = q.x; v[c][1] = q.y; v[c][2] = q.z; v[c][3] = q.w;
                } else {
                    const float4 q = __ldg(reinterpret_cast<const float4*>(p + c * plane));
                    v[c][0] = q.x; v[c][1] = q.y; v[c][2] = q.z; v[c][3] = q.w;
                }
            }
#pragma unroll
            for (int c = 0; c < 3; ++c)
#pragma unroll
                for (int j = 0; j < 4; ++j) v[c][j] = (v[c][j] - mean[c]) / stdv[c];
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (x0 + j < w) {
#pragma unroll
                    for (int c = 0; c < 3; ++c) v[c][j] = (static_cast<float>(p[c * plane + j]) - mean[c]) / stdv[c];
                }
            }
        }
    }
    __nv_bfloat16* d = dst + (static_cast<size_t>(b * Hp + y) * Wp + x0) * 4;
    if (x0 + 3 < Wp) {
        uint4 o0, o1;
        o0.x = pack2_act(v[0][0], v[1][0], fp16); o0.y = pack2_act(v[2][0], 0.f, fp16);
        o0.z = pack2_act(v[0][1], v[1][1], fp16); o0.w = pack2_act(v[2][1], 0.f, fp16);
        o1.x = pack2_act(v[0][2], v[1][2], fp16); o1.y = pack2_act(v[2][2], 0.f, fp16);
        o1.z = pack2_act(v[0][3], v[1][3], fp16); o1.w = pack2_act(v[2][3], 0.f, fp16);
        reinterpret_cast<uint4*>(d)[0] = o0;
        reinterpret_cast<uint4*>(d)[1] = o1;
    } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (x0 + j < Wp) {
                uint2 o;
                o.x = pack2_act(v[0][j], v[1][j], fp16);
                o.y = pack2_act(v[2][j], 0.f, fp16);
                reinterpret_cast<uint2*>(d)[j] = o;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------ max-pool
// element-wise maximum of 8 packed 16-bit values (paired HMNMX2 of the storage type; the flag is warp-uniform)
__device__ __forceinline__ uint4 max8(uint4 a, uint4 b, int fp16) {
    uint4 r;
    if (fp16) {
        const __half2* pa = reinterpret_cast<const __half2*>(&a);
        const __half2* pb = reinterpret_cast<const __half2*>(&b);
        __half2* pr = reinterpret_cast<__half2*>(&r);
#pragma unroll
        for (int i = 0; i < 4; ++i) pr[i] = __hmax2(pa[i], pb[i]);
    } else {
        const __nv_bfloat162* pa = reinterpret_cast<const __nv_bfloat162*>(&a);
        const __nv_bfloat162* pb = reinterpret_cast<const __nv_bfloat162*>(&b);
        __nv_bfloat162* pr = reinterpret_cast<__nv_bfloat162*>(&r);
#pragma unroll
        for (int i = 0; i < 4; ++i) pr[i] = __hmax2(pa[i], pb[i]);
    }
    return r;
}

__global__ void maxpool_kernel(const __nv_bfloat16* __restrict__ in, __nv_bfloat16* __restrict__ out, int B, int H, int W,
                               int C, int in_pitch, int Ho, int Wo, int out_pitch, int ksize, int fp16) {
    DD3D_PDL_PROLOGUE();
    const int vc = C >> 3;
    const size_t total = static_cast<size_t>(B) * Ho * Wo * vc;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int v = static_cast<int>(i % vc);
        size_t pix = i / vc;
        const int ox = static_cast<int>(pix % Wo);
        pix /= Wo;
        const int oy = static_cast<int>(pix % Ho);
        const int b = static_cast<int>(pix / Ho);
        uint4 m;
        bool first = true;
        for (int dy = 0; dy < ksize; ++dy) {
            const int iy = oy * 2 + dy;
            if (iy >= H) break;  // ceil_mode: windows are clipped to the input
            for (int dx = 0; dx < ksize; ++dx) {
                const int ix = ox * 2 + dx;
                if (ix >= W) break;
                const uint4 x = __ldg(reinterpret_cast<const uint4*>(
                    in + (static_cast<size_t>(b * H + iy) * W + ix) * in_pitch + v * 8));
                m = first ? x : max8(m, x, fp16);
                first = false;
            }
        }
        *reinterpret_cast<uint4*>(out + (static_cast<size_t>(b * Ho + oy) * Wo + ox) * out_pitch + v * 8) = m;
    }
}

// ------------------------------------------------------------------------------------------ eSE
// partial[b][split][c] = sum over the split's pixels (fixed order -> deterministic).
__global__ void ese_pool_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ partial, int HW, int C,
                                int pitch, int nsplit, int rows, int fp16) {
    DD3D_PDL_PROLOGUE();
    extern __shared__ float red[];  // [rows][C]
    const int vc = C >> 3;
    const int b = blockIdx.y, split = blockIdx.x;
    const int v = threadIdx.x % vc, r = threadIdx.x / vc;
    const int per = (HW + nsplit - 1) / nsplit;
    const int p0 = split * per, p1 = min(HW, p0 + per);
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (r < rows) {
        for (int p = p0 + r; p < p1; p += rows) {
            const uint4 u =
                __ldg(reinterpret_cast<const uint4*>(x + (static_cast<size_t>(b) * HW + p) * pitch + v * 8));
            const float2 a = unpack2_act(u.x, fp16), c = unpack2_act(u.y, fp16), d = unpack2_act(u.z, fp16), e = unpack2_act(u.w, fp16);
            acc[0] += a.x; acc[1] += a.y; acc[2] += c.x; acc[3] += c.y;
            acc[4] += d.x; acc[5] += d.y; acc[6] += e.x; acc[7] += e.y;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) red[r * C + v * 8 + j] = acc[j];
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float s = 0.f;
        for (int rr = 0; rr < rows; ++rr) s += red[rr * C + c];
        partial[(static_cast<size_t>(b) * nsplit + split) * C + c] = s;
    }
}

// sums[b][c] = sum over the T per-tile/per-warp partial rows written by the concat-conv epilogue (fixed order).
__global__ void ese_reduce_kernel(const float* __restrict__ tile_partial, float* __restrict__ sums, int T, int C,
                                  int pitch) {
    DD3D_PDL_PROLOGUE();
    __shared__ float red[4][64];
    const int b = blockIdx.y;
    const int c = blockIdx.x * 64 + (threadIdx.x & 63);
    const int grp = threadIdx.x >> 6;  // 4 row groups
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
    if (c < C) {
        const float* p = tile_partial + static_cast<size_t>(b) * T * pitch + c;
        int t = grp;
        for (; t + 12 < T; t += 16) {
            s0 += p[static_cast<size_t>(t) * pitch];
            s1 += p[static_cast<size_t>(t + 4) * pitch];
            s2 += p[static_cast<size_t>(t + 8) * pitch];
            s3 += p[static_cast<size_t>(t + 12) * pitch];
        }
        for (; t < T; t += 4) s0 += p[static_cast<size_t>(t) * pitch];
    }
    red[grp][threadIdx.x & 63] = (s0 + s1) + (s2 + s3);
    __syncthreads();
    if (grp == 0 && c < C)
        sums[static_cast<size_t>(b) * C + c] = (red[0][threadIdx.x] + red[1][threadIdx.x]) + (red[2][threadIdx.x] + red[3][threadIdx.x]);
}

// gate[b][co] = relu6(W[co,:] . mean[b,:] + bias[co] + 3) / 6      (one warp per output channel)
__global__ void ese_fc_kernel(const float* __restrict__ partial, const float* __restrict__ w, const float* __restrict__ bias,
                              float* __restrict__ gate, int C, int nsplit, float inv_hw) {
    DD3D_PDL_PROLOGUE();
    extern __shared__ float mean[];  // [C]
    const int b = blockIdx.y;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float s = 0.f;
        for (int k = 0; k < nsplit; ++k) s += partial[(static_cast<size_t>(b) * nsplit + k) * C + c];
        mean[c] = s * inv_hw;
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int co = blockIdx.x * (blockDim.x >> 5) + warp;
    if (co >= C) return;
    float s = 0.f;
    for (int ci = lane; ci < C; ci += 32) s = fmaf(w[static_cast<size_t>(co) * C + ci], mean[ci], s);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) {
        const float y = s + bias[co] + 3.0f;
        gate[static_cast<size_t>(b) * C + co] = fminf(fmaxf(y, 0.f), 6.f) / 6.0f;
    }
}

// out = 16-bit(x * gate[b][c] (+ identity)).  Pure streaming (2-3 tensor passes): every thread keeps kEseUnroll
// independent 16-byte loads of x (and of the identity) in flight per iteration -- one load per thread left the kernel at
// 66 % of the HBM roof (BENCH_r01).
constexpr int kEseUnroll = 4;
__global__ void __launch_bounds__(256) ese_scale_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ gate,
                                                        const __nv_bfloat16* __restrict__ identity,
                                                        __nv_bfloat16* __restrict__ out, int B, int HW, int C, int x_pitch,
                                                        int id_pitch, int out_pitch, int fp16) {
    DD3D_PDL_PROLOGUE();
    const int vc = C >> 3;
    const size_t total = static_cast<size_t>(B) * HW * vc;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i0 = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i0 < total; i0 += stride * kEseUnroll) {
        uint4 u[kEseUnroll], q[kEseUnroll];
        size_t pix[kEseUnroll];
        int v[kEseUnroll];
#pragma unroll
        for (int k = 0; k < kEseUnroll; ++k) {
            const size_t i = i0 + k * stride;
            v[k] = static_cast<int>(i % vc);
            pix[k] = i / vc;
            if (i < total) {
                u[k] = __ldg(reinterpret_cast<const uint4*>(x + pix[k] * x_pitch + v[k] * 8));
                if (identity != nullptr) q[k] = __ldg(reinterpret_cast<const uint4*>(identity + pix[k] * id_pitch + v[k] * 8));
            }
        }
#pragma unroll
        for (int k = 0; k < kEseUnroll; ++k) {
            if (i0 + k * stride >= total) break;
            const int b = static_cast<int>(pix[k] / HW);
            const float4 g0 = __ldg(reinterpret_cast<const float4*>(gate + static_cast<size_t>(b) * C + v[k] * 8));
            const float4 g1 = __ldg(reinterpret_cast<const float4*>(gate + static_cast<size_t>(b) * C + v[k] * 8 + 4));
            float f[8];
            float2 t;
            t = unpack2_act(u[k].x, fp16); f[0] = t.x * g0.x; f[1] = t.y * g0.y;
            t = unpack2_act(u[k].y, fp16); f[2] = t.x * g0.z; f[3] = t.y * g0.w;
            t = unpack2_act(u[k].z, fp16); f[4] = t.x * g1.x; f[5] = t.y * g1.y;
            t = unpack2_act(u[k].w, fp16); f[6] = t.x * g1.z; f[7] = t.y * g1.w;
            if (identity != nullptr) {
                t = unpack2_act(q[k].x, fp16); f[0] += t.x; f[1] += t.y;
                t = unpack2_act(q[k].y, fp16); f[2] += t.x; f[3] += t.y;
                t = unpack2_act(q[k].z, fp16); f[4] += t.x; f[5] += t.y;
                t = unpack2_act(q[k].w, fp16); f[6] += t.x; f[7] += t.y;
            }
            uint4 o;
            o.x = pack2_act(f[0], f[1], fp16); o.y = pack2_act(f[2], f[3], fp16); o.z = pack2_act(f[4], f[5], fp16);
            o.w = pack2_act(f[6], f[7], fp16);
            *reinterpret_cast<uint4*>(out + pix[k] * out_pitch + v[k] * 8) = o;
        }
    }
}

// relu on packed 16-bit floats: a set sign bit (negative, -0) -> +0; identical for bf16 and fp16
__global__ void relu_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ out, size_t nvec) {
    DD3D_PDL_PROLOGUE();
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < nvec;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        uint4 u = __ldg(reinterpret_cast<const uint4*>(x) + i);
        uint32_t* p = reinterpret_cast<uint32_t*>(&u);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint32_t neg = p[j] & 0x80008000u;             // sign bits of the two halves
            p[j] &= ~(((neg >> 15) * 0xFFFFu));                   // 0x8000 -> 0xFFFF mask per half
        }
        reinterpret_cast<uint4*>(out)[i] = u;
    }
}

inline int grid_for(size_t total, int block, int num_sms) {
    size_t g = (total + block - 1) / block;
    size_t cap = static_cast<size_t>(num_sms) * 8;
    return static_cast<int>(g < cap ? (g ? g : 1) : cap);
}

}  // namespace

cudaError_t launch_preprocess(const void* src, int src_is_u8, const int* d_sizes, int size_stride, __nv_bfloat16* dst,
                              int B, int Hs, int Ws, int Hp, int Wp, const float mean[3], const float std[3],
                              cudaStream_t stream, int fp16) {
    dim3 block(256), grid((Wp + 1023) / 1024, Hp, B);
    const int esz = src_is_u8 ? 1 : 4;
    const int vec_ok = (Ws % 4 == 0) && (reinterpret_cast<uintptr_t>(src) % (4 * esz) == 0) &&
                       ((static_cast<size_t>(Hs) * Ws) % 4 == 0);
    if (src_is_u8)
        return launch_pdl(preprocess_kernel<uint8_t>, grid, block, 0, stream, static_cast<const uint8_t*>(src), d_sizes, dst, B,
                          Hs, Ws, Hp, Wp, size_stride, mean[0], mean[1], mean[2], std[0], std[1], std[2], fp16, vec_ok);
    return launch_pdl(preprocess_kernel<float>, grid, block, 0, stream, static_cast<const float*>(src), d_sizes, dst, B, Hs, Ws,
                      Hp, Wp, size_stride, mean[0], mean[1], mean[2], std[0], std[1], std[2], fp16, vec_ok);
}

cudaError_t launch_maxpool(const __nv_bfloat16* in, __nv_bfloat16* out, int B, int H, int W, int C, int in_pitch,
                           int Ho, int Wo, int out_pitch, int ksize, int num_sms, cudaStream_t stream, int fp16) {
    const size_t total = static_cast<size_t>(B) * Ho * Wo * (C / 8);
    return launch_pdl(maxpool_kernel, dim3(grid_for(total, 256, num_sms)), dim3(256), 0, stream, in, out, B, H, W, C, in_pitch, Ho,
                      Wo, out_pitch, ksize, fp16);
}

int ese_nsplit(int HW) {
    int n = HW / 512;
    if (n < 1) n = 1;
    if (n > 64) n = 64;
    return n;
}

namespace {
// the scale pass shared by both eSE forms
cudaError_t launch_ese_scale(const __nv_bfloat16* x, int x_pitch, const float* gate, const __nv_bfloat16* identity, int id_pitch,
                             __nv_bfloat16* out, int out_pitch, int B, int HW, int C, int num_sms, cudaStream_t stream, int fp16) {
    const size_t total = static_cast<size_t>(B) * HW * (C / 8);
    return launch_pdl(ese_scale_kernel, dim3(grid_for((total + kEseUnroll - 1) / kEseUnroll, 256, num_sms)), dim3(256), 0, stream, x,
                      gate, identity, out, B, HW, C, x_pitch, id_pitch, out_pitch, fp16);
}
}  // namespace

cudaError_t launch_ese(const __nv_bfloat16* x, int x_pitch, const float* fc_w, const float* fc_b,
                       const __nv_bfloat16* identity, int id_pitch, __nv_bfloat16* out, int out_pitch, float* partial,
                       float* gate, int B, int HW, int C, int num_sms, cudaStream_t stream, int fp16) {
    const int vc = C / 8;
    int rows = 256 / vc;
    if (rows < 1) rows = 1;
    const int nsplit = ese_nsplit(HW);
    cudaError_t e = launch_pdl(ese_pool_kernel, dim3(nsplit, B), dim3(vc * rows), static_cast<size_t>(rows) * C * sizeof(float),
                               stream, x, partial, HW, C, x_pitch, nsplit, rows, fp16);
    if (e != cudaSuccess) return e;
    e = launch_pdl(ese_fc_kernel, dim3((C + 7) / 8, B), dim3(256), C * sizeof(float), stream, static_cast<const float*>(partial),
                   fc_w, fc_b, gate, C, nsplit, 1.0f / static_cast<float>(HW));
    if (e != cudaSuccess) return e;
    return launch_ese_scale(x, x_pitch, gate, identity, id_pitch, out, out_pitch, B, HW, C, num_sms, stream, fp16);
}

// eSE with the pooling partials produced by the conv epilogue: reduce -> fc -> scale (2 tensor passes instead of 3)
cudaError_t launch_ese_fused(const __nv_bfloat16* x, int x_pitch, const float* tile_partial, int T, const float* fc_w,
                             const float* fc_b, const __nv_bfloat16* identity, int id_pitch, __nv_bfloat16* out,
                             int out_pitch, float* sums, float* gate, int B, int HW, int C, int num_sms,
                             cudaStream_t stream, int fp16) {
    cudaError_t e = launch_pdl(ese_reduce_kernel, dim3((C + 63) / 64, B), dim3(256), 0, stream, tile_partial, sums, T, C, C);
    if (e != cudaSuccess) return e;
    e = launch_pdl(ese_fc_kernel, dim3((C + 7) / 8, B), dim3(256), C * sizeof(float), stream, static_cast<const float*>(sums), fc_w,
                   fc_b, gate, C, 1, 1.0f / static_cast<float>(HW));
    if (e != cudaSuccess) return e;
    return launch_ese_scale(x, x_pitch, gate, identity, id_pitch, out, out_pitch, B, HW, C, num_sms, stream, fp16);
}

cudaError_t launch_relu(const __nv_bfloat16* x, __nv_bfloat16* out, size_t n_elems, int num_sms, cudaStream_t stream) {
    const size_t nvec = n_elems / 8;
    return launch_pdl(relu_kernel, dim3(grid_for(nvec, 256, num_sms)), dim3(256), 0, stream, x, out, nvec);
}

}  // namespace dd3d
