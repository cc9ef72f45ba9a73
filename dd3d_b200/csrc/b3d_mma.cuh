// Register-fragment arithmetic shared by the two sparse FCOS3D predictors (b3d_sparse.cu, b3d_gather.cu).  An output channel
// of either kernel is the fp32 sum of the same mma.sync m16n8k16 steps over the same K order -- (tap, 64-channel block), then
// two 32-channel groups of two k16 steps each -- with the same channel permutation on both operands.  That is what makes a
// class-gathered value equal the sparse predictor's column bit for bit, so both kernels take these steps from here.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace dd3d {
namespace b3d_mma {

constexpr int kChunk = 64;  // channels per shared-memory weight block

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

__device__ __forceinline__ uint4 lds128(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
    return v;
}

// Shared-memory weight block layout of both kernels: row n of 128 bytes (64 channels), 16-byte chunk k at k ^ ((n & 1) << 2)
// (the two rows a quarter-warp reads with one LDS.128 then sit in different halves of the 128-byte line: conflict-free).
__device__ __forceinline__ uint32_t weight_slot(int n, int k) { return n * 128 + ((k ^ ((n & 1) << 2)) << 4); }

// The lane's A fragments of K block `chunk` = (tap, kc): for its two rows h (rows g and g + 8 of the warp's 16), the 16-byte
// loads of channels kc * 64 + G * 32 + 8t .. +7 of the pixel at tap offset (dy, dx); zero outside the map or for an invalid
// row.  base[h] points to channel 8t of the row's own pixel.
__device__ __forceinline__ void load_a(const __nv_bfloat16* const (&base)[2], const int (&py)[2], const int (&px)[2],
                                       const bool (&valid)[2], int H, int W, int pitch, int kcs, int chunk,
                                       uint4 (&a)[2][2]) {
    const int tap = chunk / kcs, kc = chunk - tap * kcs;
    const int dy = tap / 3 - 1, dx = tap % 3 - 1;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const bool ok = valid[h] && (py[h] + dy) >= 0 && (py[h] + dy) < H && (px[h] + dx) >= 0 && (px[h] + dx) < W;
        const __nv_bfloat16* src = base[h] + (static_cast<ptrdiff_t>(dy) * W + dx) * pitch + kc * kChunk;
#pragma unroll
        for (int G = 0; G < 2; ++G)
            a[G][h] = ok ? __ldg(reinterpret_cast<const uint4*>(src + G * 32)) : make_uint4(0u, 0u, 0u, 0u);
    }
}

// One 32-channel group G of a K block against n-tile row n (= nt * 8 + g) of the staged weights at `wb`: lane t holds
// channels 8t .. 8t+7 for its rows (lo: row g, hi: row g + 8) and for weight row n; two K = 16 steps whose k slots
// {2t, 2t+1 | 2t+8, 2t+9} are the register pairs (x, y) and (z, w) of those 16-byte loads -- the same channel permutation on
// both operands, so the products pair up correctly.
template <bool FP16>
__device__ __forceinline__ void mma_group(float (&acc)[4], const uint4& lo, const uint4& hi, uint32_t wb, int n, int G, int t) {
    const uint4 w = lds128(wb + weight_slot(n, (G << 2) | t));
    mma16816<FP16>(acc, lo.x, hi.x, lo.y, hi.y, w.x, w.y);
    mma16816<FP16>(acc, lo.z, hi.z, lo.w, hi.w, w.z, w.w);
}

}  // namespace b3d_mma
}  // namespace dd3d
