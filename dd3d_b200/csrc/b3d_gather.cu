// Class-gathered sparse FCOS3D predictor: the fused [quat | ctr | depth | size | conf] 3x3 conv of the box3d tower (reference
// fcos3d.py:102-135, per-level Scale / Offset folded into the epilogue) evaluated at the final 2-D candidates only, and for
// each candidate only at the 11 output channels {q * C + c} of its own class c -- the only ones the reference's decode reads
// (fcos3d.py:333-352).  b3d_sparse.cu keeps all 11 C channels of a row in registers, which stops at the 10 nuScenes classes;
// this kernel's work does not grow with C: a V2-99 step at PRE_NMS_TOPK 1000 is ~12 GFLOP at any class count, where the dense
// predictor at C = 128 would be 26.6 TFLOP and 23 GB of fp32 maps.
//
// Two launches:
//   1. b3d_group_kernel, one CTA per (image, level): a counting sort of the final candidates by class -> `order` (slots of
//      each class contiguous) and `seg` (first entry, count) per class.  The order inside a class is not fixed (shared-memory
//      atomics); nothing depends on it: every row is computed on its own and written to its own slot.
//   2. b3d_sparse_kernel_gathered, one CTA per (class, level, image): 8 warps x 16 candidates of that class against the 16-row
//      weight slab {q * C + c : q < 11} (5 zero rows), 74 KB in bf16 at cin 256.  The arithmetic is b3d_sparse_kernel's:
//      mma.sync m16n8k16 with fp32 accumulation, a K loop over 9 x cin / 64 blocks in (tap, 64-channel block) order, the same
//      k permutation on both operands, the same fmaf epilogue.  An output channel depends only on its activation row and its
//      weight row, so each gathered value equals column q * C + c of b3d_sparse_kernel's row bit for bit.
// Output: fp32 rows [(b * L + l) * topk + slot][kB3dGatherPitch], channel q at column q; decode_final_kernel reads them through
// DecodeParams::b3d_by_class as if the 3-D head were class agnostic.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "b3d_mma.cuh"
#include "b3d_sparse.cuh"
#include "pdl.cuh"

namespace dd3d {

namespace {

constexpr int kRowsPerCta = 128, kThreads = 256, kGroupThreads = 256;
using b3d_mma::kChunk;  // channels per shared-memory weight block
using b3d_mma::smem_u32;
using b3d_mma::weight_slot;
constexpr int kSlabRows = 16, kOutputs = 11;

// 16-byte cp.async; src_bytes 0 fills the destination with zeros (the slab's padding rows)
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}

// weight block `chunk` = (tap, kc) of class c's slab -> smem [16 rows][128 B]; slab row q < 11 is predictor row q * C3 + c,
// rows 11..15 are zero.  Layout b3d_mma::weight_slot, as in b3d_sparse.cu.
__device__ __forceinline__ void stage_slab(const __nv_bfloat16* w, int C, int c, int kcs, int chunk, uint32_t dst) {
    const int cin = kcs * kChunk, tap = chunk / kcs, kc = chunk - tap * kcs;
    if (threadIdx.x < kSlabRows * 8) {
        const int n = threadIdx.x >> 3, q = threadIdx.x & 7;
        const bool real = n < kOutputs;
        const __nv_bfloat16* src = w + static_cast<size_t>(real ? n * C + c : 0) * (9 * cin) + tap * cin + kc * kChunk + q * 8;
        cp_async16(dst + weight_slot(n, q), src, real ? 16 : 0);
    }
}

// One CTA per (image, level): counting sort of the final candidates by class.
__global__ void __launch_bounds__(kGroupThreads) b3d_group_kernel(const B3dGatherParams p) {
    DD3D_PDL_PROLOGUE();
    __shared__ int s_cnt[kB3dGatherMaxC], s_pos[kB3dGatherMaxC];
    const int bl = blockIdx.y * p.num_levels + blockIdx.x;
    const int count = min(p.cand_count[bl], p.topk);
    const uint2* fin = p.fin + static_cast<size_t>(bl) * p.topk;
    for (int c = threadIdx.x; c < p.C; c += blockDim.x) s_cnt[c] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < count; i += blockDim.x) atomicAdd(&s_cnt[fin[i].y % static_cast<uint32_t>(p.C)], 1);
    __syncthreads();
    if (threadIdx.x == 0) {
        int acc = 0;
        for (int c = 0; c < p.C; ++c) {
            s_pos[c] = acc;
            p.seg[static_cast<size_t>(bl) * p.C + c] = make_int2(acc, s_cnt[c]);
            acc += s_cnt[c];
        }
    }
    __syncthreads();
    int32_t* order = p.order + static_cast<size_t>(bl) * p.topk;
    for (int i = threadIdx.x; i < count; i += blockDim.x) order[atomicAdd(&s_pos[fin[i].y % static_cast<uint32_t>(p.C)], 1)] = i;
}

// One CTA per (class c, level l, image b): every candidate of class c at (b, l), 128 per pass.  KCS as in b3d_sparse.cu.
template <bool FP16, int KCS>
__global__ void __launch_bounds__(kThreads) b3d_sparse_kernel_gathered(const B3dGatherParams p) {
    DD3D_PDL_PROLOGUE();
    extern __shared__ __align__(16) uint8_t smem[];
    const int c = blockIdx.x, l = blockIdx.y, b = blockIdx.z;
    const int bl = b * p.num_levels + l;
    const int2 sg = p.seg[static_cast<size_t>(bl) * p.C + c];
    if (sg.y == 0) return;  // block-uniform
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int kcs = KCS > 0 ? KCS : p.cin / kChunk, chunks = 9 * kcs;
    const uint32_t s_w = smem_u32(smem);
    constexpr uint32_t buf_bytes = kSlabRows * 128;
    const B3dSparseLevel& L = p.lvl[l];
    const int32_t* order = p.order + static_cast<size_t>(bl) * p.topk + sg.x;

    for (int r0 = 0; r0 < sg.y; r0 += kRowsPerCta) {
        // the two rows of this lane's fragments: candidate -> pixel -> pointer to channel 8t of the tap (0, 0) pixel
        const __nv_bfloat16* base[2];
        int py[2], px[2], slot[2];
        bool valid[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = r0 + warp * 16 + g + 8 * h;
            valid[h] = row < sg.y;
            slot[h] = valid[h] ? order[row] : 0;
            const uint32_t idx = valid[h] ? p.fin[static_cast<size_t>(bl) * p.topk + slot[h]].y : 0u;
            const int pix = static_cast<int>(idx / static_cast<uint32_t>(p.C));
            py[h] = pix / L.W;
            px[h] = pix - py[h] * L.W;
            base[h] = L.in + (static_cast<size_t>(b * L.H + py[h]) * L.W + px[h]) * L.pitch + 8 * t;
        }
        auto load_a = [&](int chunk, uint4 (&a)[2][2]) {  // [group of 32 channels][row half]
            b3d_mma::load_a(base, py, px, valid, L.H, L.W, L.pitch, kcs, chunk, a);
        };

        float acc[2][4];
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[nt][j] = 0.f;

        uint4 a_cur[2][2], a_nxt[2][2];
        stage_slab(L.w, p.C, c, kcs, 0, s_w);
        asm volatile("cp.async.commit_group;" ::: "memory");
        load_a(0, a_cur);
        for (int k = 0; k < chunks; ++k) {
            if (k + 1 < chunks) {
                stage_slab(L.w, p.C, c, kcs, k + 1, s_w + ((k + 1) & 1) * buf_bytes);
                load_a(k + 1, a_nxt);
            }
            asm volatile("cp.async.commit_group;" ::: "memory");
            asm volatile("cp.async.wait_group 1;" ::: "memory");
            __syncthreads();  // weight block k is in shared memory
            const uint32_t wb = s_w + (k & 1) * buf_bytes;
#pragma unroll
            for (int G = 0; G < 2; ++G)
#pragma unroll
                for (int nt = 0; nt < 2; ++nt) b3d_mma::mma_group<FP16>(acc[nt], a_cur[G][0], a_cur[G][1], wb, nt * 8 + g, G, t);
            __syncthreads();  // every warp is done with buffer k & 1 before block k + 2 is staged into it
#pragma unroll
            for (int G = 0; G < 2; ++G)
#pragma unroll
                for (int h = 0; h < 2; ++h) a_cur[G][h] = a_nxt[G][h];
        }
        asm volatile("cp.async.wait_group 0;" ::: "memory");

        // epilogue: y = acc * scale + bias of predictor channel q * C + c, written to column q of the candidate's row
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const int q = nt * 8 + 2 * t + j;
                if (q < kOutputs) {
                    const int ch = q * p.C + c;
                    const float s = __ldg(L.scale + ch), bb = __ldg(L.bias + ch);
#pragma unroll
                    for (int h = 0; h < 2; ++h)
                        if (valid[h])
                            p.rows[(static_cast<size_t>(bl) * p.topk + slot[h]) * kB3dGatherPitch + q] = fmaf(acc[nt][2 * h + j], s, bb);
                }
            }
        }
    }
}

template <int KCS>
cudaError_t launch_gathered(const B3dGatherParams& p, cudaStream_t stream) {
    constexpr int smem = 2 * kSlabRows * 128;
    const dim3 grid(p.C, p.num_levels, p.B);
    if (p.fp16) return launch_pdl(b3d_sparse_kernel_gathered<true, KCS>, grid, dim3(kThreads), smem, stream, p);
    return launch_pdl(b3d_sparse_kernel_gathered<false, KCS>, grid, dim3(kThreads), smem, stream, p);
}

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

}  // namespace

size_t b3d_gather_scratch_bytes(int B, int C, int topk, int num_levels) {
    const size_t bl = static_cast<size_t>(B) * num_levels;
    return align_up(bl * topk * 4, 256) + align_up(bl * C * 8, 256);
}

void b3d_gather_bind_scratch(B3dGatherParams* p, void* scratch) {
    const size_t bl = static_cast<size_t>(p->B) * p->num_levels;
    uint8_t* s = static_cast<uint8_t*>(scratch);
    p->order = reinterpret_cast<int32_t*>(s);
    p->seg = reinterpret_cast<int2*>(s + align_up(bl * p->topk * 4, 256));
}

cudaError_t launch_b3d_gather(const B3dGatherParams& p, cudaStream_t stream) {
    if (p.B < 1 || p.topk < 1 || p.C < 1 || p.C > kB3dGatherMaxC || p.order == nullptr || p.seg == nullptr)
        return cudaErrorInvalidValue;
    if (p.cin < kChunk || p.cin % kChunk || p.cin > kB3dSparseMaxCin) return cudaErrorInvalidValue;
    if (p.num_levels < 1 || p.num_levels > kLevels) return cudaErrorInvalidValue;
    for (int l = 0; l < p.num_levels; ++l)
        if (p.lvl[l].pitch % 8 || p.lvl[l].pitch < p.cin || p.lvl[l].in == nullptr || p.lvl[l].w == nullptr ||
            p.lvl[l].scale == nullptr || p.lvl[l].bias == nullptr)
            return cudaErrorInvalidValue;
    cudaError_t e = launch_pdl(b3d_group_kernel, dim3(p.num_levels, p.B), dim3(kGroupThreads), 0, stream, p);
    if (e != cudaSuccess) return e;
    return p.cin == 256 ? launch_gathered<4>(p, stream) : launch_gathered<0>(p, stream);
}

}  // namespace dd3d
