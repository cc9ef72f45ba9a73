// Depthwise 3x3 convolution (VoVNet -dw variants: dw_conv3x3, reference vovnet.py:100-121): groups = C, padding 1,
// stride 1 or 2, no bias / norm / activation (the pointwise 1x1 that follows carries pw_norm + ReLU and runs on the
// implicit-GEMM conv).  NHWC 16-bit views with a channel pitch; weights 16-bit [9][C] (tap-major, tap = r * 3 + s).
//
// One CTA = one TH x TW output tile of one image for one 64-channel slice.  The input tile plus its one-pixel halo is
// staged in shared memory with 16-byte cp.async; pixels outside the view are stored as zeros, which is the conv padding.
// Each thread owns one 8-channel vector and a few output pixels of the tile, keeps its 9 x 8 weights in registers and
// accumulates in fp32 in a fixed tap order (r-major, then s), rounding once at the store -> bit-deterministic.
#include "act16.cuh"
#include "pdl.cuh"
#include "small_kernels.cuh"

namespace dd3d {

namespace {

constexpr int kDwThreads = 256;
constexpr int kDwSlice = 64;  // channels per CTA
constexpr int kDwVecs = kDwSlice / 8;

template <int STRIDE>
struct DwTile {
    static constexpr int TH = 8;
    static constexpr int TW = STRIDE == 1 ? 16 : 8;
    static constexpr int IH = (TH - 1) * STRIDE + 3;
    static constexpr int IW = (TW - 1) * STRIDE + 3;
};

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
    const uint32_t s = static_cast<uint32_t>(__cvta_generic_to_shared(smem));
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gmem) : "memory");
}

template <int STRIDE>
__global__ void __launch_bounds__(kDwThreads) dwconv3x3_kernel(const __nv_bfloat16* __restrict__ in, int H, int W, int C,
                                                                int in_pitch, const __nv_bfloat16* __restrict__ w,
                                                                __nv_bfloat16* __restrict__ out, int Ho, int Wo, int out_pitch,
                                                                int tiles_x, int tiles_per_image, int fp16) {
    DD3D_PDL_PROLOGUE();
    using T = DwTile<STRIDE>;
    __shared__ __align__(16) uint4 patch[T::IH * T::IW * kDwVecs];
    const int tile = blockIdx.x % tiles_per_image, b = blockIdx.x / tiles_per_image;
    const int oy0 = (tile / tiles_x) * T::TH, ox0 = (tile % tiles_x) * T::TW;
    const int c0 = blockIdx.y * kDwSlice;
    const int nv = min(kDwVecs, (C - c0) >> 3);  // 8-channel vectors of this slice
    const int iy0 = oy0 * STRIDE - 1, ix0 = ox0 * STRIDE - 1;
    const __nv_bfloat16* img = in + static_cast<size_t>(b) * H * W * in_pitch + c0;
    for (int i = threadIdx.x; i < T::IH * T::IW * kDwVecs; i += kDwThreads) {
        const int v = i % kDwVecs, px = i / kDwVecs;
        const int iy = iy0 + px / T::IW, ix = ix0 + px % T::IW;
        if (v >= nv) continue;
        if (iy >= 0 && iy < H && ix >= 0 && ix < W)
            cp_async16(&patch[i], img + (static_cast<size_t>(iy) * W + ix) * in_pitch + v * 8);
        else
            patch[i] = make_uint4(0u, 0u, 0u, 0u);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    const int v = threadIdx.x % kDwVecs;
    float wf[9][8];
    if (v < nv) {
#pragma unroll
        for (int t = 0; t < 9; ++t) {
            const uint4 u = __ldg(reinterpret_cast<const uint4*>(w + static_cast<size_t>(t) * C + c0 + v * 8));
            const float2 a = unpack2_act(u.x, fp16), bb = unpack2_act(u.y, fp16), c = unpack2_act(u.z, fp16),
                         d = unpack2_act(u.w, fp16);
            wf[t][0] = a.x; wf[t][1] = a.y; wf[t][2] = bb.x; wf[t][3] = bb.y;
            wf[t][4] = c.x; wf[t][5] = c.y; wf[t][6] = d.x; wf[t][7] = d.y;
        }
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    if (v >= nv) return;
    __nv_bfloat16* dst = out + static_cast<size_t>(b) * Ho * Wo * out_pitch + c0 + v * 8;
    for (int p = threadIdx.x / kDwVecs; p < T::TH * T::TW; p += kDwThreads / kDwVecs) {
        const int ty = p / T::TW, tx = p % T::TW;
        const int oy = oy0 + ty, ox = ox0 + tx;
        if (oy >= Ho || ox >= Wo) continue;
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int s = 0; s < 3; ++s) {
                const uint4 u = patch[((ty * STRIDE + r) * T::IW + tx * STRIDE + s) * kDwVecs + v];
                const float2 a = unpack2_act(u.x, fp16), bb = unpack2_act(u.y, fp16), c = unpack2_act(u.z, fp16),
                             d = unpack2_act(u.w, fp16);
                const float x[8] = {a.x, a.y, bb.x, bb.y, c.x, c.y, d.x, d.y};
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[j] = fmaf(x[j], wf[r * 3 + s][j], acc[j]);
            }
        uint4 o;
        o.x = pack2_act(acc[0], acc[1], fp16);
        o.y = pack2_act(acc[2], acc[3], fp16);
        o.z = pack2_act(acc[4], acc[5], fp16);
        o.w = pack2_act(acc[6], acc[7], fp16);
        *reinterpret_cast<uint4*>(dst + (static_cast<size_t>(oy) * Wo + ox) * out_pitch) = o;
    }
}

template <int STRIDE>
cudaError_t launch_dw(const __nv_bfloat16* in, int B, int H, int W, int C, int in_pitch, const __nv_bfloat16* w,
                      __nv_bfloat16* out, int out_pitch, cudaStream_t stream, int fp16) {
    using T = DwTile<STRIDE>;
    const int Ho = dwconv3x3_out_size(H, STRIDE), Wo = dwconv3x3_out_size(W, STRIDE);
    const int tiles_x = (Wo + T::TW - 1) / T::TW, tiles_y = (Ho + T::TH - 1) / T::TH;
    const long blocks = static_cast<long>(B) * tiles_x * tiles_y;
    if (blocks < 1 || blocks > 0x7fffffffL) return cudaErrorInvalidValue;
    return launch_pdl(dwconv3x3_kernel<STRIDE>, dim3(static_cast<unsigned>(blocks), (C + kDwSlice - 1) / kDwSlice),
                      dim3(kDwThreads), 0, stream, in, H, W, C, in_pitch, w, out, Ho, Wo, out_pitch, tiles_x,
                      tiles_x * tiles_y, fp16);
}

}  // namespace

int dwconv3x3_out_size(int n, int stride) { return (n - 1) / stride + 1; }

cudaError_t launch_dwconv3x3(const __nv_bfloat16* in, int B, int H, int W, int C, int in_pitch, const __nv_bfloat16* w,
                             int stride, __nv_bfloat16* out, int out_pitch, cudaStream_t stream, int fp16) {
    if (B < 1 || H < 1 || W < 1 || C < 8 || C % 8 || in_pitch % 8 || out_pitch % 8 || in_pitch < C || out_pitch < C)
        return cudaErrorInvalidValue;
    if (reinterpret_cast<uintptr_t>(in) % 16 || reinterpret_cast<uintptr_t>(out) % 16 || reinterpret_cast<uintptr_t>(w) % 16)
        return cudaErrorInvalidValue;
    if (stride == 1) return launch_dw<1>(in, B, H, W, C, in_pitch, w, out, out_pitch, stream, fp16);
    if (stride == 2) return launch_dw<2>(in, B, H, W, C, in_pitch, w, out, out_pitch, stream, fp16);
    return cudaErrorInvalidValue;
}

}  // namespace dd3d
