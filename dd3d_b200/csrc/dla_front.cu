// DLA-34 front end in ONE kernel: base_layer (7x7, 3->16) -> level0 (3x3, 16->16) -> level1 (3x3 stride 2, 16->32), each
// conv + FrozenBN + ReLU (reference dla.py:271-283 `base_layer`, `level0`, `level1`, forward dla.py:346-350), plus the 2x2
// max-pool of level1's output that level2's Tree takes as `bottom` (dla.py:235).
//
// Why a separate kernel.  The three layers carry 4 % of DLA-34's FLOPs but, run one by one, a large share of the forward
// (B = 8, 384x1280): each writes and re-reads a full-resolution 16-channel map (126 MB) and none has enough K (<= 16 per
// tap) or N (<= 32) for a wgmma tile -- a 64x16 A tile costs the same shared-memory read whatever N is, and the
// taps-in-N form pays a 576 B/pixel fp32 round trip through shared memory.  Here the two full-resolution intermediates
// never leave the SM: a CTA owns an 8x32 tile of level1's output, recomputes the 19x67 / 17x65 halo regions of base_layer /
// level0 in shared memory and writes only level1 (+ its pooled copy).  HBM traffic per image pixel: 8 B in, 16 B + 4 B out
// (was 8 + 32 + 32 + 32 + 16 + 16 + 4).
//
// Arithmetic: warp-level mma.sync.m16n8k16 (bf16 or fp16 operands, fp32 accumulate) on purpose -- the operand fragments
// are gathered straight from the shared-memory patches (LDS.64 of whole input pixels for the 7x7, ldmatrix of 16-channel
// pixels for the 3x3s, any shift / stride for free), the accumulators live in registers and the BN + ReLU + 16-bit
// rounding happens there, so there is no im2col copy, no shared-memory round trip of the accumulators and no CTA-wide
// barrier inside a layer.  The kernel is bound by shared-memory wavefronts and the mma.sync path, not by HBM or wgmma peak.
//
// Numerics are those of the layer-by-layer path (and of the oracle's 16-bit emulation): every intermediate is rounded to
// the storage type, conv padding is zero OUTSIDE THE IMAGE (halo positions beyond the border are forced to 0 after the
// epilogue, they are not "the conv evaluated out there").
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>

#include "act16.cuh"
#include "device_once.cuh"
#include "small_kernels.cuh"

namespace dd3d {

namespace {

constexpr int T1H = 8, T1W = 32;                    // level1 output tile (256 pixels)
constexpr int R0H = 2 * T1H + 1, R0W = 2 * T1W + 1;  // level0 region feeding it: 17 x 65
constexpr int RBH = R0H + 2, RBW = R0W + 2;          // base_layer region: 19 x 67
// input region: 25 x 74.  One column more than the 7x7 window needs: the K padding column (kx = 7, zero weights) of the
// rightmost pixels reads it, and 0 x (whatever shared memory held) must stay finite
constexpr int IH = RBH + 6, IW = RBW + 7;
constexpr int R0PX = R0H * R0W, RBPX = RBH * RBW, IPX = IH * IW;
constexpr int kInBytes = (IPX * 8 + 15) / 16 * 16;  // one input patch (4 x 16 bit per pixel)
constexpr int kBaseBytes = RBPX * 32;               // 16 channels x 16 bit per pixel, 16-byte halves XOR-swizzled
constexpr int kL0Bytes = R0PX * 32;
constexpr int kSmemBytes = 2 * kInBytes + kBaseBytes + kL0Bytes;
constexpr int kThreads = 256, kWarps = kThreads / 32;
static_assert(T1H == kWarps, "level1 phase: one warp per (row pair, half row)");
static_assert(kBaseBytes >= kWarps * 2 * 16 * 64, "output staging aliases the base_layer patch");

struct FrontParams {
    const __nv_bfloat16* in;   // [B][H][W][4] normalised image (4th channel 0)
    const __nv_bfloat16* w0;   // base_layer [16][7][8][4]  (kx = 7 and c = 3 zero)
    const __nv_bfloat16* w1;   // level0 [16][9][16]
    const __nv_bfloat16* w2;   // level1 [32][9][16]
    const float* sb0;          // scale[16] | bias[16]
    const float* sb1;          // scale[16] | bias[16]
    const float* sb2;          // scale[32] | bias[32]
    __nv_bfloat16* out;        // level1 [B][H/2][W/2][out_pitch]
    __nv_bfloat16* pool;       // 2x2 max-pool of it [B][H/4][W/4][pool_pitch] (nullptr: none)
    int B, H, W, H1, W1, out_pitch, pool_pitch, tiles_x, tiles_y;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

template <bool FP16>
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    if (FP16) {
        asm volatile(
            "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    } else {
        asm volatile(
            "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    }
}

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(addr));
}
__device__ __forceinline__ uint2 lds64(uint32_t addr) {
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts32(uint32_t addr, uint32_t v) {
    asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void cp_async8(uint32_t dst, const void* src, uint32_t src_bytes) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}

template <bool FP16>
__device__ __forceinline__ uint32_t pack2(float a, float b) {
    return FP16 ? pack2_f16(a, b) : pack2_bf16(a, b);
}
template <bool FP16>
__device__ __forceinline__ uint32_t max2(uint32_t a, uint32_t b) {
    if (FP16) {
        __half2 r = __hmax2(*reinterpret_cast<__half2*>(&a), *reinterpret_cast<__half2*>(&b));
        return *reinterpret_cast<uint32_t*>(&r);
    }
    __nv_bfloat162 r = __hmax2(*reinterpret_cast<__nv_bfloat162*>(&a), *reinterpret_cast<__nv_bfloat162*>(&b));
    return *reinterpret_cast<uint32_t*>(&r);
}
template <bool FP16>
__device__ __forceinline__ uint4 max8(uint4 a, uint4 b) {
    return make_uint4(max2<FP16>(a.x, b.x), max2<FP16>(a.y, b.y), max2<FP16>(a.z, b.z), max2<FP16>(a.w, b.w));
}

// byte offset of the 16-byte half `half` (channels 8*half .. 8*half+7) of pixel `px` in a 32 B/pixel patch.  The XOR with
// bit 2 of the pixel index makes 8 consecutive pixels (ldmatrix rows, epilogue rows g and g+4) hit 8 distinct bank groups.
__device__ __forceinline__ uint32_t px_off(int px, int half) { return static_cast<uint32_t>(px * 32 + ((half ^ ((px >> 2) & 1)) << 4)); }

__device__ __forceinline__ void tile_coords(const FrontParams& p, int tile, int* b, int* oy0, int* ox0) {
    const int per = p.tiles_x * p.tiles_y;
    *b = tile / per;
    const int r = tile - *b * per;
    const int ty = r / p.tiles_x;
    *oy0 = ty * T1H;
    *ox0 = (r - ty * p.tiles_x) * T1W;
}

// asynchronous copy of the 25 x 74 input patch of `tile` (zero-filled outside the image)
__device__ __forceinline__ void load_input(const FrontParams& p, int tile, uint32_t dst) {
    int b, oy0, ox0;
    tile_coords(p, tile, &b, &oy0, &ox0);
    const int iy0 = 2 * oy0 - 5, ix0 = 2 * ox0 - 5;
    const __nv_bfloat16* img = p.in + static_cast<size_t>(b) * p.H * p.W * 4;
    // warp -> patch rows, lane -> columns: no integer division in the address math
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
__global__ void __launch_bounds__(kThreads, 2) dla_front_kernel(const FrontParams p) {
    extern __shared__ __align__(16) uint8_t smem[];
    const uint32_t s_in = smem_u32(smem);
    const uint32_t s_base = s_in + 2 * kInBytes;
    const uint32_t s_l0 = s_base + kBaseBytes;
    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
    const int g = lane >> 2, t = lane & 3;
    // ldmatrix.x4 role of this lane: it supplies the address of row `lm_row` (0..15), k-half `lm_half`
    const int lm_row = (lane & 7) + ((lane >> 3) & 1) * 8, lm_half = lane >> 4;
    const int total = p.B * p.tiles_x * p.tiles_y;

    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

    int tile = blockIdx.x;
    if (tile < total) load_input(p, tile, s_in);
    asm volatile("cp.async.commit_group;" ::: "memory");
    int buf = 0;
    for (; tile < total; tile += gridDim.x, buf ^= 1) {
        const int next = tile + gridDim.x;
        if (next < total) load_input(p, next, s_in + (buf ^ 1) * kInBytes);
        asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_group 1;" ::: "memory");
        __syncthreads();  // this tile's input patch is complete and visible; the previous tile's phases are all done

        int b, oy0, ox0;
        tile_coords(p, tile, &b, &oy0, &ox0);
        const uint32_t s_cur = s_in + buf * kInBytes;

        // ---------------------------------------------------------------- base_layer: 7x7, 3(+1) -> 16, over 19 x 67
        {
            // B fragments.  K step ks = ky*2 + h covers input pixels kx = 4h .. 4h+3 of kernel row ky; inside a step the
            // mma k index is mapped so that lane t's four k values {2t, 2t+1, 2t+8, 2t+9} are the four channels of pixel
            // kx = 4h + t: one LDS.64 per fragment row on the A side, one 8-byte load per (step, n-tile) here.
            uint2 wb[14][2];
#pragma unroll
            for (int ks = 0; ks < 14; ++ks)
#pragma unroll
                for (int nt = 0; nt < 2; ++nt)
                    wb[ks][nt] = __ldg(reinterpret_cast<const uint2*>(p.w0) + (nt * 8 + g) * 56 + ks * 4 + t);
            float sc[2][2], bi[2][2];
#pragma unroll
            for (int nt = 0; nt < 2; ++nt)
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    sc[nt][j] = __ldg(p.sb0 + nt * 8 + 2 * t + j);
                    bi[nt][j] = __ldg(p.sb0 + 16 + nt * 8 + 2 * t + j);
                }
            const int by0 = 2 * oy0 - 2, bx0 = 2 * ox0 - 2;  // image coordinates of the region's origin
            for (int mt = warp; mt < (RBPX + 15) / 16; mt += kWarps) {
                const int p_lo = mt * 16 + g, p_hi = p_lo + 8;
                const int q_lo = min(p_lo, RBPX - 1), q_hi = min(p_hi, RBPX - 1);
                const int y_lo = q_lo / RBW, x_lo = q_lo - y_lo * RBW;
                const int y_hi = q_hi / RBW, x_hi = q_hi - y_hi * RBW;
                const uint32_t a_lo = s_cur + (y_lo * IW + x_lo + t) * 8;
                const uint32_t a_hi = s_cur + (y_hi * IW + x_hi + t) * 8;
                float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
#pragma unroll
                for (int ks = 0; ks < 14; ++ks) {
                    const uint32_t off = ((ks >> 1) * IW + (ks & 1) * 4) * 8;
                    const uint2 lo = lds64(a_lo + off), hi = lds64(a_hi + off);
                    const uint32_t a[4] = {lo.x, hi.x, lo.y, hi.y};
                    mma16816<FP16>(acc[0], a, wb[ks][0].x, wb[ks][0].y);
                    mma16816<FP16>(acc[1], a, wb[ks][1].x, wb[ks][1].y);
                }
                const bool in_lo = (by0 + y_lo) >= 0 && (by0 + y_lo) < p.H && (bx0 + x_lo) >= 0 && (bx0 + x_lo) < p.W;
                const bool in_hi = (by0 + y_hi) >= 0 && (by0 + y_hi) < p.H && (bx0 + x_hi) >= 0 && (bx0 + x_hi) < p.W;
#pragma unroll
                for (int nt = 0; nt < 2; ++nt) {
                    const uint32_t v_lo = pack2_relu<FP16>(fmaf(acc[nt][0], sc[nt][0], bi[nt][0]), fmaf(acc[nt][1], sc[nt][1], bi[nt][1]));
                    const uint32_t v_hi = pack2_relu<FP16>(fmaf(acc[nt][2], sc[nt][0], bi[nt][0]), fmaf(acc[nt][3], sc[nt][1], bi[nt][1]));
                    if (p_lo < RBPX) sts32(s_base + px_off(p_lo, nt) + t * 4, in_lo ? v_lo : 0u);
                    if (p_hi < RBPX) sts32(s_base + px_off(p_hi, nt) + t * 4, in_hi ? v_hi : 0u);
                }
            }
        }
        __syncthreads();

        // ---------------------------------------------------------------- level0: 3x3, 16 -> 16, over 17 x 65
        {
            uint32_t wb[9][2][2];
#pragma unroll
            for (int tap = 0; tap < 9; ++tap)
#pragma unroll
                for (int nt = 0; nt < 2; ++nt) {
                    const uint32_t* w = reinterpret_cast<const uint32_t*>(p.w1 + ((nt * 8 + g) * 9 + tap) * 16);
                    wb[tap][nt][0] = __ldg(w + t);
                    wb[tap][nt][1] = __ldg(w + 4 + t);
                }
            float sc[2][2], bi[2][2];
#pragma unroll
            for (int nt = 0; nt < 2; ++nt)
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    sc[nt][j] = __ldg(p.sb1 + nt * 8 + 2 * t + j);
                    bi[nt][j] = __ldg(p.sb1 + 16 + nt * 8 + 2 * t + j);
                }
            const int ly0 = 2 * oy0 - 1, lx0 = 2 * ox0 - 1;
            for (int mt = warp; mt < (R0PX + 15) / 16; mt += kWarps) {
                const int q = min(mt * 16 + lm_row, R0PX - 1);
                const int qy = q / R0W, qx = q - qy * R0W;
                const int pb0 = qy * RBW + qx;  // base-region pixel under tap (0, 0)
                float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
#pragma unroll
                for (int tap = 0; tap < 9; ++tap) {
                    uint32_t a[4];
                    ldmatrix_x4(a, s_base + px_off(pb0 + (tap / 3) * RBW + (tap % 3), lm_half));
                    mma16816<FP16>(acc[0], a, wb[tap][0][0], wb[tap][0][1]);
                    mma16816<FP16>(acc[1], a, wb[tap][1][0], wb[tap][1][1]);
                }
                const int p_lo = mt * 16 + g, p_hi = p_lo + 8;
                const int y_lo = p_lo / R0W, x_lo = p_lo - y_lo * R0W;
                const int y_hi = p_hi / R0W, x_hi = p_hi - y_hi * R0W;
                const bool in_lo = (ly0 + y_lo) >= 0 && (ly0 + y_lo) < p.H && (lx0 + x_lo) >= 0 && (lx0 + x_lo) < p.W;
                const bool in_hi = (ly0 + y_hi) >= 0 && (ly0 + y_hi) < p.H && (lx0 + x_hi) >= 0 && (lx0 + x_hi) < p.W;
#pragma unroll
                for (int nt = 0; nt < 2; ++nt) {
                    const uint32_t v_lo = pack2_relu<FP16>(fmaf(acc[nt][0], sc[nt][0], bi[nt][0]), fmaf(acc[nt][1], sc[nt][1], bi[nt][1]));
                    const uint32_t v_hi = pack2_relu<FP16>(fmaf(acc[nt][2], sc[nt][0], bi[nt][0]), fmaf(acc[nt][3], sc[nt][1], bi[nt][1]));
                    if (p_lo < R0PX) sts32(s_l0 + px_off(p_lo, nt) + t * 4, in_lo ? v_lo : 0u);
                    if (p_hi < R0PX) sts32(s_l0 + px_off(p_hi, nt) + t * 4, in_hi ? v_hi : 0u);
                }
            }
        }
        __syncthreads();

        // ---------------------------------------------------------------- level1: 3x3 stride 2, 16 -> 32, 8 x 32 outputs
        {
            uint32_t wb[9][4][2];
#pragma unroll
            for (int tap = 0; tap < 9; ++tap)
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) {
                    const uint32_t* w = reinterpret_cast<const uint32_t*>(p.w2 + ((nt * 8 + g) * 9 + tap) * 16);
                    wb[tap][nt][0] = __ldg(w + t);
                    wb[tap][nt][1] = __ldg(w + 4 + t);
                }
            // this warp: output rows 2*(warp/2), 2*(warp/2)+1, columns 16*(warp%2) .. +15 -> it also owns the 8 pooled
            // pixels under them.  Staging (16-bit results, 64 B per pixel) aliases the base_layer patch, which is dead.
            const int row0 = 2 * (warp >> 1), col0 = 16 * (warp & 1);
            const uint32_t s_stage = s_base + warp * (2 * 16 * 64);
#pragma unroll
            for (int m = 0; m < 2; ++m) {
                const int oy = row0 + m;
                const int pl0 = (2 * oy) * R0W + 2 * (col0 + lm_row);  // level0-region pixel under tap (0, 0)
                float acc[4][4];
#pragma unroll
                for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                    for (int j = 0; j < 4; ++j) acc[nt][j] = 0.f;
#pragma unroll
                for (int tap = 0; tap < 9; ++tap) {
                    uint32_t a[4];
                    ldmatrix_x4(a, s_l0 + px_off(pl0 + (tap / 3) * R0W + (tap % 3), lm_half));
#pragma unroll
                    for (int nt = 0; nt < 4; ++nt) mma16816<FP16>(acc[nt], a, wb[tap][nt][0], wb[tap][nt][1]);
                }
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) {
                    const float s0 = __ldg(p.sb2 + nt * 8 + 2 * t), s1 = __ldg(p.sb2 + nt * 8 + 2 * t + 1);
                    const float b0 = __ldg(p.sb2 + 32 + nt * 8 + 2 * t), b1 = __ldg(p.sb2 + 32 + nt * 8 + 2 * t + 1);
                    const uint32_t v_lo = pack2_relu<FP16>(fmaf(acc[nt][0], s0, b0), fmaf(acc[nt][1], s1, b1));
                    const uint32_t v_hi = pack2_relu<FP16>(fmaf(acc[nt][2], s0, b0), fmaf(acc[nt][3], s1, b1));
                    // pixel (m, x): 64 B, its four 16-byte chunks XOR-swizzled by (x >> 1) & 3 (rows g / g+2 / g+4 / g+6
                    // would otherwise share banks)
                    sts32(s_stage + (m * 16 + g) * 64 + ((nt ^ ((g >> 1) & 3)) << 4) + t * 4, v_lo);
                    sts32(s_stage + (m * 16 + g + 8) * 64 + ((nt ^ (((g + 8) >> 1) & 3)) << 4) + t * 4, v_hi);
                }
            }
            __syncwarp();
            // coalesced 16-byte stores: 2 rows x 16 pixels x 4 chunks = 128 chunks, 4 per lane
            const int gy0 = oy0 + row0, gx0 = ox0 + col0;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int c = j * 32 + lane;
                const int m = c >> 6, x = (c >> 2) & 15, ch = c & 3;
                const uint4 v = lds128(s_stage + (m * 16 + x) * 64 + ((ch ^ ((x >> 1) & 3)) << 4));
                if (gy0 + m < p.H1 && gx0 + x < p.W1)
                    *reinterpret_cast<uint4*>(p.out + (static_cast<size_t>(b * p.H1 + gy0 + m) * p.W1 + gx0 + x) * p.out_pitch + ch * 8) = v;
            }
            if (p.pool != nullptr) {  // 2x2 / stride 2 max-pool of the two rows: 8 pooled pixels x 4 chunks = one per lane
                const int px = lane >> 2, ch = lane & 3;
                const int xa = 2 * px, xb = 2 * px + 1;
                const uint32_t oa = ((ch ^ ((xa >> 1) & 3)) << 4), ob = ((ch ^ ((xb >> 1) & 3)) << 4);
                uint4 v = max8<FP16>(lds128(s_stage + xa * 64 + oa), lds128(s_stage + xb * 64 + ob));
                v = max8<FP16>(v, max8<FP16>(lds128(s_stage + (16 + xa) * 64 + oa), lds128(s_stage + (16 + xb) * 64 + ob)));
                const int H2 = p.H1 >> 1, W2 = p.W1 >> 1;
                const int py = gy0 >> 1, pxg = (gx0 >> 1) + px;
                if (py < H2 && pxg < W2)
                    *reinterpret_cast<uint4*>(p.pool + (static_cast<size_t>(b * H2 + py) * W2 + pxg) * p.pool_pitch + ch * 8) = v;
            }
        }
        // no barrier here: the next iteration's __syncthreads (after its input wait) orders this tile's reads of the
        // level0 patch / staging before the next tile's writes
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
}

}  // namespace

// Packed weight sizes (16-bit elements): base_layer [16][7][8][4], level0 [16][9][16], level1 [32][9][16].
cudaError_t launch_dla_front(const __nv_bfloat16* in4, const __nv_bfloat16* w0, const __nv_bfloat16* w1,
                             const __nv_bfloat16* w2, const float* sb0, const float* sb1, const float* sb2,
                             __nv_bfloat16* out, int out_pitch, __nv_bfloat16* pool, int pool_pitch, int B, int H, int W,
                             int num_sms, cudaStream_t stream, int fp16) {
    if (H % 2 || W % 2 || out_pitch % 8 || (pool != nullptr && (pool_pitch % 8 || H % 4 || W % 4))) return cudaErrorInvalidValue;
    FrontParams p;
    p.in = in4; p.w0 = w0; p.w1 = w1; p.w2 = w2; p.sb0 = sb0; p.sb1 = sb1; p.sb2 = sb2;
    p.out = out; p.pool = pool;
    p.B = B; p.H = H; p.W = W; p.H1 = H / 2; p.W1 = W / 2;
    p.out_pitch = out_pitch; p.pool_pitch = pool_pitch;
    p.tiles_x = (p.W1 + T1W - 1) / T1W;
    p.tiles_y = (p.H1 + T1H - 1) / T1H;
    static uint64_t attr_devices[2] = {0, 0};
    if (first_use_on_device(&attr_devices[fp16 ? 1 : 0])) {
        cudaError_t e = fp16 ? cudaFuncSetAttribute(dla_front_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes)
                             : cudaFuncSetAttribute(dla_front_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
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
    return fp16 ? cudaLaunchKernelEx(&cfg, dla_front_kernel<true>, p) : cudaLaunchKernelEx(&cfg, dla_front_kernel<false>, p);
}

}  // namespace dd3d
