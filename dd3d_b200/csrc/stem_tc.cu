// Stem convolutions (Cin = 3) on Hopper tensor cores (wgmma).
//
// Replaces DLA `base_layer` (7x7 s1, 3->16, reference dla.py:271-280) and VoVNet `stem_1` (3x3 s2, 3->64,
// vovnet.py:302) + FrozenBN + ReLU.  Cin=3 is too thin for TMA-fed implicit GEMM (a pixel is 8 bytes), so the CTA
// builds the im2col tile itself: thread m gathers the KSxKS neighbourhood of output pixel m from the normalised
// bf16 [B][H][W][4] image (4th channel = 0) and writes it as one K-major, 128B-swizzled operand row
// (k = (ky*KS + kx)*4 + c), then the warpgroup issues the wgmmas (two M = 64 halves of the 128 pixels, N = Cout, K padded
// to 16) and runs the epilogue from its accumulator registers.  Several CTAs per SM overlap gather / MMA / epilogue of
// different tiles.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>

#include "act16.cuh"
#include "device_once.cuh"
#include "ptx.cuh"
#include "small_kernels.cuh"
#include "wgmma.cuh"

namespace dd3d {

namespace {

constexpr int kTileH = 8, kTileW = 16;  // 128 output pixels
constexpr int kStemThreads = 128;       // one warpgroup

template <int KS, int STRIDE, int COUT, bool F16>
__global__ void __launch_bounds__(kStemThreads) stem_tc_kernel(const __nv_bfloat16* __restrict__ in, const __nv_bfloat16* __restrict__ w,
                                                               const float* __restrict__ scale, const float* __restrict__ bias,
                                                               __nv_bfloat16* __restrict__ out, int B, int H, int W, int Ho, int Wo,
                                                               int out_pitch, int tiles_x, int tiles_y, int relu) {
    constexpr int PAD = (KS - 1) / 2;
    constexpr int K = KS * KS * 4;            // 36 / 196
    constexpr int KB = (K + 63) / 64;         // 64-element k-blocks: 1 / 4
    constexpr int KSTEPS = (K + 15) / 16;     // wgmma K=16 steps: 3 / 13
    constexpr int CHUNKS = (KS * KS + 1) / 2; // 16-byte chunks (2 taps each) per row that carry data
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sA = smem;                     // [KB][128 rows][128 B]
    uint8_t* sB = smem + KB * 16384;        // [KB][COUT rows][128 B]
    __shared__ __align__(16) float s_scale[COUT];  // folded BN, read as broadcast LDS in the epilogue
    __shared__ __align__(16) float s_bias[COUT];
    const uint32_t sA_u32 = ptx::smem_u32(sA);     // explicit STS: the integer-aligned pointer would compile to generic ST.E
    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    // weights -> swizzled smem (global layout [COUT][KB*64] bf16, K contiguous)
    for (int i = tid; i < COUT * KB * 8; i += blockDim.x) {
        const int n = i / (KB * 8), q = i - n * (KB * 8);
        const int kb = q >> 3, c = q & 7;
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(w + static_cast<size_t>(n) * KB * 64) + q);
        *reinterpret_cast<uint4*>(sB + kb * COUT * 128 + n * 128 + ((c ^ (n & 7)) << 4)) = v;
    }
    // zero the K padding of the operand rows once (chunks >= CHUNKS never change)
    for (int q = CHUNKS; q < KB * 8; ++q)
        ptx::st_shared_v4(sA_u32 + (q >> 3) * 16384 + tid * 128 + (((q & 7) ^ (tid & 7)) << 4), make_uint4(0, 0, 0, 0));
    for (int i = tid; i < COUT; i += blockDim.x) {
        s_scale[i] = __ldg(scale + i);
        s_bias[i] = __ldg(bias + i);
    }
    __syncthreads();
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

    const uint64_t desc_hi = ptx::make_sw128_desc(0) & ~0x3FFFull;
    const uint32_t a_lo = ptx::smem_u32(sA) >> 4;
    const uint32_t b_lo = ptx::smem_u32(sB) >> 4;
    const int total = B * tiles_x * tiles_y;
    for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
        const int b = tile / (tiles_x * tiles_y);
        const int r = tile - b * tiles_x * tiles_y;
        const int ty = r / tiles_x, tx = r - ty * tiles_x;
        {
            // ---- im2col gather: one operand row per thread
            const int oy = ty * kTileH + (tid >> 4), ox = tx * kTileW + (tid & 15);
            const int iy0 = oy * STRIDE - PAD, ix0 = ox * STRIDE - PAD;
            const __nv_bfloat16* img = in + static_cast<size_t>(b) * H * W * 4;
            // fully unrolled: all KS*KS predicated 8-byte loads are issued before the first use (memory-level
            // parallelism instead of one load latency per tap)
            uint2 v[KS * KS + 1];
#pragma unroll
            for (int ky = 0; ky < KS; ++ky) {
                const int iy = iy0 + ky;
                const bool rok = (iy >= 0) && (iy < H);
                const __nv_bfloat16* rowp = img + (static_cast<ptrdiff_t>(iy) * W + ix0) * 4;
#pragma unroll
                for (int kx = 0; kx < KS; ++kx) {
                    const int ix = ix0 + kx;
                    v[ky * KS + kx] = make_uint2(0u, 0u);
                    if (rok && ix >= 0 && ix < W) v[ky * KS + kx] = __ldg(reinterpret_cast<const uint2*>(rowp + kx * 4));
                }
            }
            v[KS * KS] = make_uint2(0u, 0u);
#pragma unroll
            for (int q = 0; q < CHUNKS; ++q)
                ptx::st_shared_v4(sA_u32 + (q >> 3) * 16384 + tid * 128 + (((q & 7) ^ (tid & 7)) << 4),
                                  make_uint4(v[2 * q].x, v[2 * q].y, v[2 * q + 1].x, v[2 * q + 1].y));
            ptx::fence_proxy_async_smem();  // generic-proxy writes -> visible to the tensor core (async proxy)
        }
        __syncthreads();
        // ---- two M = 64 halves of the tile, N = COUT
        float acc[2][COUT / 2];
        wg::fence();
#pragma unroll
        for (int m = 0; m < 2; ++m) {
#pragma unroll
            for (int s = 0; s < KSTEPS; ++s) {
                const int kb = s >> 2, k = s & 3;
                const uint64_t adesc = desc_hi | (a_lo + kb * (16384 >> 4) + m * (64 * 128 >> 4) + 2 * k);
                const uint64_t bdesc = desc_hi | (b_lo + kb * ((COUT * 128) >> 4) + 2 * k);
                wg::wgmma<COUT, F16>(acc[m], adesc, bdesc, s > 0 ? 1u : 0u);
            }
        }
        wg::commit();
        wg::wait<0>();
        wg::fence_regs(acc[0]);
        wg::fence_regs(acc[1]);
        // ---- epilogue: scale/bias/ReLU -> bf16 -> global.  d[4j + 2h + e] = (row 16 warp + lane/4 + 8h, col 8j + 2(lane%4) + e)
#pragma unroll
        for (int m = 0; m < 2; ++m) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int pix = 64 * m + 16 * warp + (lane >> 2) + 8 * h;
                const int oy = ty * kTileH + (pix >> 4), ox = tx * kTileW + (pix & 15);
                if (oy < Ho && ox < Wo) {
                    __nv_bfloat16* dst = out + (static_cast<size_t>(b * Ho + oy) * Wo + ox) * out_pitch + 2 * (lane & 3);
#pragma unroll
                    for (int j = 0; j < COUT / 8; ++j) {
                        const int col = 8 * j + 2 * (lane & 3);
                        float y0 = fmaf(acc[m][4 * j + 2 * h], s_scale[col], s_bias[col]);
                        float y1 = fmaf(acc[m][4 * j + 2 * h + 1], s_scale[col + 1], s_bias[col + 1]);
                        if (relu) {  // 0: the raw output a GroupNorm normalises
                            y0 = fmaxf(y0, 0.f);
                            y1 = fmaxf(y1, 0.f);
                        }
                        *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack2_act(y0, y1, F16 ? 1 : 0);
                    }
                }
            }
        }
        __syncthreads();  // operand tile consumed before the next tile overwrites it
    }
}

template <int KS, int STRIDE, int COUT>
cudaError_t launch_one(const __nv_bfloat16* in, const __nv_bfloat16* w, const float* scale, const float* bias,
                       __nv_bfloat16* out, int B, int H, int W, int out_pitch, int num_sms, cudaStream_t stream,
                       int fp16, int relu) {
    constexpr int PAD = (KS - 1) / 2;
    constexpr int KB = (KS * KS * 4 + 63) / 64;
    const int Ho = (H + 2 * PAD - KS) / STRIDE + 1, Wo = (W + 2 * PAD - KS) / STRIDE + 1;
    const int tiles_x = (Wo + kTileW - 1) / kTileW, tiles_y = (Ho + kTileH - 1) / kTileH;
    const int smem = KB * 16384 + KB * COUT * 128 + 1024;
    static uint64_t attr_devices = 0;  // per template instantiation, per device
    if (first_use_on_device(&attr_devices)) {
        cudaError_t e = cudaFuncSetAttribute(stem_tc_kernel<KS, STRIDE, COUT, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e == cudaSuccess)
            e = cudaFuncSetAttribute(stem_tc_kernel<KS, STRIDE, COUT, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) return e;
    }
    const int ctas_per_sm = std::max(1, std::min(4, (200 * 1024) / smem));
    const int total = B * tiles_x * tiles_y;
    const int grid = std::min(total, num_sms * ctas_per_sm);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(kStemThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return fp16 ? cudaLaunchKernelEx(&cfg, stem_tc_kernel<KS, STRIDE, COUT, true>, in, w, scale, bias, out, B, H, W, Ho, Wo,
                                     out_pitch, tiles_x, tiles_y, relu)
                : cudaLaunchKernelEx(&cfg, stem_tc_kernel<KS, STRIDE, COUT, false>, in, w, scale, bias, out, B, H, W, Ho, Wo,
                                     out_pitch, tiles_x, tiles_y, relu);
}

}  // namespace

int stem_tc_kpad(int ksize) { return (ksize * ksize * 4 + 63) / 64 * 64; }

// in: bf16 [B][H][W][4]; w: bf16 [cout][stem_tc_kpad(ksize)] with k = (ky*ksize + kx)*4 + c; out: NHWC bf16.
cudaError_t launch_stem_tc(const __nv_bfloat16* in, const __nv_bfloat16* w, const float* scale, const float* bias,
                           __nv_bfloat16* out, int B, int H, int W, int ksize, int stride, int cout, int out_pitch,
                           int num_sms, cudaStream_t stream, int fp16, int relu) {
    if (ksize == 7 && stride == 1 && cout == 16)
        return launch_one<7, 1, 16>(in, w, scale, bias, out, B, H, W, out_pitch, num_sms, stream, fp16, relu);
    if (ksize == 3 && stride == 2 && cout == 64)
        return launch_one<3, 2, 64>(in, w, scale, bias, out, B, H, W, out_pitch, num_sms, stream, fp16, relu);
    return cudaErrorInvalidValue;
}

}  // namespace dd3d
