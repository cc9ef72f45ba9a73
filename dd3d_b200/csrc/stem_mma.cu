// VoVNet stem_1 (3x3 stride 2, 3 -> 64, FrozenBN + ReLU; reference vovnet.py:302 via conv3x3 / stem, forward vovnet.py:357-359)
// as a register-fragment kernel.
//
// The layer is a pure streaming problem: 0.39 GB of normalised input in, 1.57 GB of 64-channel output out per 32-image batch
// around 75 GFLOP.  The wgmma form (stem_tc.cu) builds a K-major im2col tile in shared memory per 128 pixels
// (thread-gathered, 9 predicated 8-byte loads + swizzled stores per pixel, then wgmma).  Here a CTA copies the 17 x 66
// input patch of an 8 x 32 output tile with cp.async (double buffered), and every warp feeds mma.sync.m16n8k16 straight from it: one K step per kernel row, its 16 k slots = 4
// consecutive input pixels x 4 channels (4th pixel / 4th channel carry zero weights), so lane t's fragment registers are ONE
// 8-byte shared-memory load of input pixel 2x - 1 + t.  The 64 x 48 weight fragments stay in registers for the whole kernel.
// Output channels are PERMUTED across the n-tiles (column j of n-tile nt = channel 16 (j / 2) + 2 nt + (j % 2)) so that the
// 16 accumulator columns a lane holds for one pixel are 16 consecutive channels: BN + ReLU + rounding happen in registers and
// the results leave as two 16-byte global stores per pixel and lane -- no shared-memory staging, no shuffles.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "act16.cuh"
#include "device_once.cuh"
#include "small_kernels.cuh"

namespace dd3d {

namespace {

constexpr int TH = 8, TW = 32;                   // output tile
constexpr int IH = 2 * TH + 1, IW = 2 * TW + 2;  // input patch 17 x 66 (one spare column for the zero-weight k slot)
constexpr int kInBytes = IH * IW * 8;
constexpr int kThreads = 256, kWarps = 8;
constexpr int kBufs = 4;  // input patches in flight: a tile's math is ~700 cycles, a DRAM round trip ~2 000
constexpr int kSmemBytes = kBufs * kInBytes;
static_assert(TH * TW == kWarps * 2 * 16, "two 16-pixel M tiles per warp");

struct StemParams {
    const __nv_bfloat16* in;  // [B][H][W][4]
    const __nv_bfloat16* w;   // [64][3][4][4]: cout, ky, kx (kx = 3 zero), c (c = 3 zero)
    const float* sb;          // scale[64] | bias[64]
    __nv_bfloat16* out;       // [B][Ho][Wo][out_pitch]
    int B, H, W, Ho, Wo, out_pitch, tiles_x, tiles_y;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

template <bool FP16>
__device__ __forceinline__ void mma16816(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                         uint32_t b1) {
    if (FP16) {
        asm volatile(
            "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
            : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
    } else {
        asm volatile(
            "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
            : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
    }
}
__device__ __forceinline__ uint2 lds64(uint32_t addr) {
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr));
    return v;
}
__device__ __forceinline__ void cp_async8(uint32_t dst, const void* src, uint32_t src_bytes) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}

__device__ __forceinline__ void tile_coords(const StemParams& p, int tile, int* b, int* oy0, int* ox0) {
    const int per = p.tiles_x * p.tiles_y;
    *b = tile / per;
    const int r = tile - *b * per;
    const int ty = r / p.tiles_x;
    *oy0 = ty * TH;
    *ox0 = (r - ty * p.tiles_x) * TW;
}

__device__ __forceinline__ void load_input(const StemParams& p, int tile, uint32_t dst) {
    int b, oy0, ox0;
    tile_coords(p, tile, &b, &oy0, &ox0);
    const int iy0 = 2 * oy0 - 1, ix0 = 2 * ox0 - 1;
    const __nv_bfloat16* img = p.in + static_cast<size_t>(b) * p.H * p.W * 4;
    // warp -> patch rows, lane -> columns: no integer division in the address math (it was ~45 % of the kernel's instructions)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int y = warp; y < IH; y += kWarps) {
        const int gy = iy0 + y;
        const bool row_ok = gy >= 0 && gy < p.H;
        const __nv_bfloat16* row = img + static_cast<size_t>(row_ok ? gy : 0) * p.W * 4;
#pragma unroll
        for (int x = lane; x < IW; x += 32) {
            const int gx = ix0 + x;
            const bool ok = row_ok && gx >= 0 && gx < p.W;
            cp_async8(dst + (y * IW + x) * 8, row + (ok ? gx * 4 : 0), ok ? 8u : 0u);
        }
    }
}

template <bool FP16>
__global__ void __launch_bounds__(kThreads, 2) stem_s2_mma_kernel(const StemParams p) {
    extern __shared__ __align__(16) uint8_t smem[];
    const uint32_t s_in = smem_u32(smem);
    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
    const int g = lane >> 2, t = lane & 3;
    const int total = p.B * p.tiles_x * p.tiles_y;

    // weight fragments of all 8 n-tiles x 3 kernel rows, resident for the whole kernel: lane (g, t) holds output channel
    // 16 (g / 2) + 2 nt + (g % 2) (the column permutation above), input pixel kx = t, channels (0, 1) in b0 and (2, 3) in b1
    // -- the same k-slot mapping as the A loads below
    uint2 wb[3][8];
#pragma unroll
    for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
            wb[ky][nt] = __ldg(reinterpret_cast<const uint2*>(p.w) + ((16 * (g >> 1) + 2 * nt + (g & 1)) * 3 + ky) * 4 + t);

    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

    // kBufs-deep ring of input patches: tiles k .. k + kBufs - 2 are in flight while tile k is computed.  A buffer may be
    // refilled only after the barrier that retires its readers: the patch of tile k + kBufs - 1 goes into the buffer tile k - 1
    // was read from, and is issued AFTER the barrier at the top of iteration k.
    int tile = blockIdx.x;
#pragma unroll
    for (int i = 0; i < kBufs - 1; ++i) {
        const int tl = tile + i * static_cast<int>(gridDim.x);
        if (tl < total) load_input(p, tl, s_in + i * kInBytes);
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    int buf = 0;
    for (; tile < total; tile += gridDim.x, buf = (buf + 1) % kBufs) {
        asm volatile("cp.async.wait_group %0;" ::"n"(kBufs - 2) : "memory");  // all but the newest kBufs - 2 groups: tile k landed
        __syncthreads();  // ... and is visible to all warps, and every warp has finished tile k - 1
        const int ahead = tile + (kBufs - 1) * static_cast<int>(gridDim.x);
        if (ahead < total) load_input(p, ahead, s_in + ((buf + kBufs - 1) % kBufs) * kInBytes);
        asm volatile("cp.async.commit_group;" ::: "memory");
        int b, oy0, ox0;
        tile_coords(p, tile, &b, &oy0, &ox0);
        const uint32_t s_cur = s_in + buf * kInBytes;
#pragma unroll 1
        for (int m = 0; m < 2; ++m) {
            // M tile = 16 consecutive output pixels of one tile row: row = warp, columns 16 m .. 16 m + 15
            const int oy = warp, oxl = 16 * m;
            const uint32_t a_lo = s_cur + ((2 * oy) * IW + 2 * (oxl + g) + t) * 8;
            const uint32_t a_hi = a_lo + 16 * 8;  // output pixel + 8 -> input pixel + 16
            float acc[8][4];
#pragma unroll
            for (int nt = 0; nt < 8; ++nt)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[nt][j] = 0.f;
#pragma unroll
            for (int ky = 0; ky < 3; ++ky) {
                const uint2 lo = lds64(a_lo + ky * IW * 8), hi = lds64(a_hi + ky * IW * 8);
#pragma unroll
                for (int nt = 0; nt < 8; ++nt) mma16816<FP16>(acc[nt], lo.x, hi.x, lo.y, hi.y, wb[ky][nt].x, wb[ky][nt].y);
            }
            // BN + ReLU + rounding in registers: this lane's columns are channels 16 t .. 16 t + 15 of rows g and g + 8
            uint32_t o_lo[8], o_hi[8];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float4 sc = __ldg(reinterpret_cast<const float4*>(p.sb + 16 * t) + q);
                const float4 bi = __ldg(reinterpret_cast<const float4*>(p.sb + 64 + 16 * t) + q);
                o_lo[2 * q] = pack2_relu<FP16>(fmaf(acc[2 * q][0], sc.x, bi.x), fmaf(acc[2 * q][1], sc.y, bi.y));
                o_hi[2 * q] = pack2_relu<FP16>(fmaf(acc[2 * q][2], sc.x, bi.x), fmaf(acc[2 * q][3], sc.y, bi.y));
                o_lo[2 * q + 1] = pack2_relu<FP16>(fmaf(acc[2 * q + 1][0], sc.z, bi.z), fmaf(acc[2 * q + 1][1], sc.w, bi.w));
                o_hi[2 * q + 1] = pack2_relu<FP16>(fmaf(acc[2 * q + 1][2], sc.z, bi.z), fmaf(acc[2 * q + 1][3], sc.w, bi.w));
            }
            const int gy = oy0 + oy;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int gx = ox0 + oxl + g + 8 * h;
                if (gy < p.Ho && gx < p.Wo) {
                    const uint32_t* o = h ? o_hi : o_lo;
                    __nv_bfloat16* dst = p.out + (static_cast<size_t>(b * p.Ho + gy) * p.Wo + gx) * p.out_pitch + 16 * t;
                    reinterpret_cast<uint4*>(dst)[0] = make_uint4(o[0], o[1], o[2], o[3]);
                    reinterpret_cast<uint4*>(dst)[1] = make_uint4(o[4], o[5], o[6], o[7]);
                }
            }
        }
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
}

}  // namespace

// in4: [B][H][W][4]; w: 16-bit [64][3][4][4] (cout, ky, kx, c; kx = 3 and c = 3 zero); sb: fp32 scale[64] | bias[64];
// out: [B][ceil(H/2)][ceil(W/2)][out_pitch].
cudaError_t launch_stem_s2_mma(const __nv_bfloat16* in4, const __nv_bfloat16* w, const float* sb, __nv_bfloat16* out,
                               int out_pitch, int B, int H, int W, int num_sms, cudaStream_t stream, int fp16) {
    if (out_pitch % 8 || B < 1 || H < 1 || W < 1) return cudaErrorInvalidValue;
    StemParams p;
    p.in = in4; p.w = w; p.sb = sb; p.out = out;
    p.B = B; p.H = H; p.W = W; p.Ho = (H + 1) / 2; p.Wo = (W + 1) / 2;
    p.out_pitch = out_pitch;
    p.tiles_x = (p.Wo + TW - 1) / TW;
    p.tiles_y = (p.Ho + TH - 1) / TH;
    static uint64_t attr_devices[2] = {0, 0};
    if (first_use_on_device(&attr_devices[fp16 ? 1 : 0])) {
        cudaError_t e = fp16 ? cudaFuncSetAttribute(stem_s2_mma_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes)
                             : cudaFuncSetAttribute(stem_s2_mma_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
        if (e != cudaSuccess) return e;
    }
    const int total = B * p.tiles_x * p.tiles_y;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(std::min(total, 2 * num_sms));
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = kSmemBytes;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return fp16 ? cudaLaunchKernelEx(&cfg, stem_s2_mma_kernel<true>, p) : cudaLaunchKernelEx(&cfg, stem_s2_mma_kernel<false>, p);
}

}  // namespace dd3d
