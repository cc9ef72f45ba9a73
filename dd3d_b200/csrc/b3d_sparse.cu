// Sparse FCOS3D predictor: the fused [quat | ctr | depth | size | conf] 3x3 conv of the box3d tower (reference fcos3d.py:
// 102-135 `box3d_quat/ctr/depth/size/conf`, applied in forward fcos3d.py:160-188, per-level Scale / Offset folded into the
// epilogue) evaluated ONLY at the pixels that survived the 2-D threshold + per-level top-k (fcos2d.py:280-310) -- the 3-D
// outputs of every other pixel are never read by the reference's inference either (fcos3d.py:328-399 indexes them with the
// 2-D candidates).  Dense, the layer is 0.53 TFLOP of a V2-99 step (32 x 127 875 pixels x 2304 x 110); the
// bench batch keeps ~1 100 candidates per image: 115 x fewer rows.
//
// Gathered GEMM: row = one final candidate (image b, level l, slot) of decode.cu's `fin` list, K = 9 taps x cin channels (the
// FPN width FE.FPN.OUT_CHANNELS: a multiple of 64, 256 by default) read straight from the NHWC tower output at the candidate's 3x3 neighbourhood (zeros outside the map), N = the fused predictor's
// output channels.  One CTA = 128 rows of one (image, level); warp = 16 rows x all N in registers (mma.sync m16n8k16, fp32
// accumulate -- the rows are gathered per lane with 16-byte loads, which is exactly the fragment layout once K is permuted
// identically on both operands; the work is ~20 GFLOP per step, the tensor path is not the limit).  The K loop runs over
// 9 x cin / 64 blocks in (tap, 64-channel block) order, so every width sums in the same order as the 256-wide layer.  The
// weight tile of a 64-channel block is staged in shared memory by cp.async (double buffered) and shared by the 8 warps.
// Output: fp32 rows [(b * L + l) * topk + slot][pitch] in the channel layout of a dense map pixel; decode_final_kernel reads
// them through DecodeParams::b3d_rows.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "b3d_mma.cuh"
#include "b3d_sparse.cuh"
#include "pdl.cuh"

namespace dd3d {

namespace {

constexpr int kRowsPerCta = 128, kThreads = 256;
using b3d_mma::kChunk;  // channels per shared-memory weight block
using b3d_mma::smem_u32;
using b3d_mma::weight_slot;

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}

// weight block `chunk` = (tap, kc) of predictor `w` ([n_pad][9][cin]) -> smem [n_pad rows][128 B] (b3d_mma::weight_slot)
__device__ __forceinline__ void stage_weights(const __nv_bfloat16* w, int n_pad, int kcs, int chunk, uint32_t dst) {
    const int cin = kcs * kChunk, tap = chunk / kcs, kc = chunk - tap * kcs;
    const __nv_bfloat16* src = w + tap * cin + kc * kChunk;
    for (int i = threadIdx.x; i < n_pad * 8; i += kThreads) {
        const int n = i >> 3, q = i & 7;
        cp_async16(dst + weight_slot(n, q), src + static_cast<size_t>(n) * (9 * cin) + q * 8);
    }
}

// KCS: 64-channel blocks per tap (cin / 64) as a compile-time constant (4: the default 256-wide FPN), or 0 to read it from
// p.cin at run time (every other width; the runtime division costs 16 registers)
template <int NT, bool FP16, int KCS>
__global__ void __launch_bounds__(kThreads) b3d_sparse_kernel(const B3dSparseParams p) {
    DD3D_PDL_PROLOGUE();
    extern __shared__ __align__(16) uint8_t smem[];
    const int b = blockIdx.z, l = blockIdx.y, r0 = blockIdx.x * kRowsPerCta;
    const int bl = b * p.num_levels + l;
    const int count = min(p.cand_count[bl], p.topk);
    if (r0 >= count) return;  // block-uniform
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int nt_real = p.n_pad >> 3;
    const int kcs = KCS > 0 ? KCS : p.cin / kChunk, chunks = 9 * kcs;
    const uint32_t s_w = smem_u32(smem);
    const uint32_t buf_bytes = static_cast<uint32_t>(p.n_pad) * 128;
    const B3dSparseLevel& L = p.lvl[l];

    // the two rows of this lane's fragments: candidate -> pixel -> pointer to channel 8t of the tap (0, 0) pixel
    const __nv_bfloat16* base[2];
    int py[2], px[2];
    bool valid[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int row = r0 + warp * 16 + g + 8 * h;
        valid[h] = row < count;
        const uint32_t idx = valid[h] ? p.fin[static_cast<size_t>(bl) * p.topk + row].y : 0u;
        const int pix = static_cast<int>(idx / static_cast<uint32_t>(p.C));
        py[h] = pix / L.W;
        px[h] = pix - py[h] * L.W;
        base[h] = L.in + (static_cast<size_t>(b * L.H + py[h]) * L.W + px[h]) * L.pitch + 8 * t;
    }
    auto load_a = [&](int chunk, uint4 (&a)[2][2]) {  // [group of 32 channels][row half]
        b3d_mma::load_a(base, py, px, valid, L.H, L.W, L.pitch, kcs, chunk, a);
    };

    float acc[NT][4];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[nt][j] = 0.f;

    uint4 a_cur[2][2], a_nxt[2][2];
    stage_weights(L.w, p.n_pad, kcs, 0, s_w);
    asm volatile("cp.async.commit_group;" ::: "memory");
    load_a(0, a_cur);
    for (int c = 0; c < chunks; ++c) {
        if (c + 1 < chunks) {
            stage_weights(L.w, p.n_pad, kcs, c + 1, s_w + ((c + 1) & 1) * buf_bytes);
            load_a(c + 1, a_nxt);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_group 1;" ::: "memory");
        __syncthreads();  // weight block c is in shared memory
        const uint32_t wb = s_w + (c & 1) * buf_bytes;
#pragma unroll
        for (int G = 0; G < 2; ++G) {
#pragma unroll
            for (int nt = 0; nt < NT; ++nt)
                if (nt < nt_real) b3d_mma::mma_group<FP16>(acc[nt], a_cur[G][0], a_cur[G][1], wb, nt * 8 + g, G, t);
        }
        __syncthreads();  // every warp is done with buffer c & 1 before block c + 2 is staged into it
#pragma unroll
        for (int G = 0; G < 2; ++G)
#pragma unroll
            for (int h = 0; h < 2; ++h) a_cur[G][h] = a_nxt[G][h];
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");

    // epilogue: y = acc * scale + bias (per-level Scale / Offset and the conv biases folded by the engine), fp32 rows
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
        if (nt < nt_real) {
            const int n0 = nt * 8 + 2 * t;
            const float s0 = __ldg(L.scale + n0), s1 = __ldg(L.scale + n0 + 1);
            const float b0 = __ldg(L.bias + n0), b1 = __ldg(L.bias + n0 + 1);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = r0 + warp * 16 + g + 8 * h;
                if (row < count) {
                    float2 v = make_float2(fmaf(acc[nt][2 * h], s0, b0), fmaf(acc[nt][2 * h + 1], s1, b1));
                    *reinterpret_cast<float2*>(p.rows + (static_cast<size_t>(bl) * p.topk + row) * p.out_pitch + n0) = v;
                }
            }
        }
    }
}

template <int NT, int KCS>
cudaError_t launch_nt(const B3dSparseParams& p, cudaStream_t stream) {
    const int smem = 2 * p.n_pad * 128;
    dim3 grid((p.topk + kRowsPerCta - 1) / kRowsPerCta, p.num_levels, p.B);
    if (p.fp16) return launch_pdl(b3d_sparse_kernel<NT, true, KCS>, grid, dim3(kThreads), smem, stream, p);
    return launch_pdl(b3d_sparse_kernel<NT, false, KCS>, grid, dim3(kThreads), smem, stream, p);
}

template <int NT>
cudaError_t launch_cin(const B3dSparseParams& p, cudaStream_t stream) {
    return p.cin == 256 ? launch_nt<NT, 4>(p, stream) : launch_nt<NT, 0>(p, stream);
}

}  // namespace

cudaError_t launch_b3d_sparse(const B3dSparseParams& p, cudaStream_t stream) {
    if (p.n_pad < 8 || p.n_pad % 8 || p.n_pad > kB3dSparseMaxN || p.out_pitch < p.n_pad || p.out_pitch % 2 || p.B < 1 || p.topk < 1)
        return cudaErrorInvalidValue;
    if (p.cin < kChunk || p.cin % kChunk || p.cin > kB3dSparseMaxCin) return cudaErrorInvalidValue;
    if (p.num_levels < 1 || p.num_levels > kLevels) return cudaErrorInvalidValue;
    for (int l = 0; l < p.num_levels; ++l)
        if (p.lvl[l].pitch % 8 || p.lvl[l].pitch < p.cin || p.lvl[l].in == nullptr || p.lvl[l].w == nullptr)
            return cudaErrorInvalidValue;
    if (p.n_pad <= 64) return launch_cin<8>(p, stream);   // C3 <= 5 (KITTI: 5 classes -> 55 -> 64), class-agnostic (11 -> 16)
    return launch_cin<14>(p, stream);                      // nuScenes: 10 classes -> 110 -> 112
}

}  // namespace dd3d
