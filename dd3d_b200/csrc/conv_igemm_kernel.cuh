// Implicit-GEMM convolution on Hopper tensor cores (sm_90a: TMA + mbarrier pipeline + wgmma).
//
// Replaces every cuDNN conv + FrozenBN/BN + ReLU (+residual, +FPN upsample-add) launch of the reference's
// DD3D.forward (SURVEY.md 2.1 K1/K2/K3/K6; reference call sites dla.py:27-46,149-157,229-231, vovnet.py:129-157,
// detectron2 FPN, fcos2d.py:81-98, fcos3d.py:90-126).
//
// GEMM view:  D[m][n] = sum_k A[m][k] * W[n][k]
//   m : 128 output pixels of one th x tw patch of one image          (two consumer warpgroups, wgmma M = 64 each)
//   n : output channels, block_n <= 256 per tile                       (wgmma N = block_n)
//   k : taps x input channels, 64 channels (128 B) per k-block         (wgmma K = 16, 4 per k-block)
// A is never materialised: for tap (r,s) the k-block is ONE tiled TMA box [1][th][tw][64ch] of the NHWC bf16
// input at spatial offset (r-1, s-1); TMA zero-fills out-of-image pixels (= conv zero padding) and channels
// beyond C (ragged C such as 160/224).  Stride-2 convs read a parity-split 5-D view of the same tensor.
// Concats are free: producers TMA-store into channel slices of one wide NHWC buffer, the 1x1 reads it whole.
//
// Halo variant (3x3, stride 1): the A operand of a 64-channel block is ONE box [18][10][64ch] (tile + halo); the nine
// taps are descriptor views of it shifted by whole 128-byte pixel rows, so A is fetched once instead of nine times.
//
// Warpgroup roles (384 threads, 1 CTA/SM, persistent over tiles); the producer loops are warp-converged and only the issue
// instructions are predicated on elect.sync, which keeps the TMA operands in uniform registers:
//   warp 0 : TMA producer of the activation tiles (generic) / of the weight tiles (halo)
//   warp 2 : TMA producer of the weight tiles (generic) / of the halo patches (halo)
//   warpgroups 1, 2 : consumers.  Warpgroup 1 + w owns tile rows 64 w .. 64 w + 63: it issues the wgmmas of its rows (fp32
//                accumulators in registers, one commit group per k-block, the smem slot of k-block i released once group
//                i + 1 is issued and group i retired), then runs the epilogue of its rows (scale/bias/residual/ReLU ->
//                bf16/fp16 -> swizzled staging tile -> TMA store, optional eSE pooling partial sums; or fp32 direct stores
//                for the predictor heads).  The producers keep prefetching the next tile's operands during the epilogue.
// Launched with programmatic dependent launch: the prologue overlaps the previous kernel's tail.
//
// Pair tile (PAIR, halo only, block_n = 128): the work item is TWO 16x8 halo tiles (tiles 2i, 2i + 1 of one image in
// row-major tile order) x one 128-channel n-block, so every weight tile fetched from L2 feeds 256 output pixels instead of
// 128 -- half the weight bytes per MAC of the 128 x 256 tile, for about 39 % less L2->SM traffic.  Warpgroup 1 + w owns
// sub-tile w (its own [18][10][64ch] patch) and issues two m64n128k16 wgmmas per K step, one per 64-row half, on the same B
// descriptor; it stores its sub-tile itself (own staging buffers, named barrier and store leader).  An odd per-image tile
// count leaves the last pair's second sub-tile outside the image: its rows are never stored and read no residual.  The K
// order per output element is unchanged, so results are bit-identical to the 128 x 256 tile.
//
// Work-list mode (LIST, pair tile only): the M units come from ConvParams::tile_list, whose length the kernel reads from the
// device after griddepcontrol.wait, so a launch can cover a tile set an earlier kernel chose (the sparse towers, engine.cu)
// without a host round trip; the grid stays persistent.  The unit is four listed 8x8 tiles (kListTile), so that a sparse tower
// computes fewer pixels around its seeds than with 16x8 tiles: warpgroup 1 + w owns tiles 2w and 2w + 1, one per 64-row
// half, each read from its own [10][10][64ch] patch (four patches per A stage, on one barrier).  The descriptor views are the
// halo tile's (row-group stride of 10 pixels, taps as whole-pixel-row shifts), the weight tile and the K order the dense pair
// tile's, so every computed pixel is bit-identical to it.  The four patches leave room for three B stages (stagger 1).
//
// The kernel is templated on (halo variant, fp16 storage, wgmma N = block_n, pair tile, work list); conv_igemm_n*.cu instantiate it, one
// group of N values per translation unit so that the build compiles them in parallel; conv_igemm.cu holds the host side and
// the taps-in-N kernel.
#pragma once
#include "conv_igemm.cuh"

#include <math.h>

#include "act16.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace dd3d {

namespace {


constexpr int kABytes = kBlockM * kBlockK * 2;  // 16 KiB
constexpr int kStagingBytes = kBlockM * 128;    // one 64-channel bf16 output chunk
constexpr int kHalfStagingBytes = kStagingBytes / 2;  // its 64 rows of one consumer warpgroup (one TMA store box)
constexpr int kMaxStages = 8;
constexpr int kSmemBudget = 227 * 1024;
// halo variant: per 64-channel block the A operand is ONE (16+2)x(8+2)-pixel patch = 180 rows of 128 B (64 channels),
// 128B-swizzled by TMA; the slot is rounded up to a multiple of 1024 B so every patch keeps the swizzle-atom alignment
constexpr int kHaloPW = kHaloTw + 2, kHaloPH = kHaloTh + 2;
constexpr int kHaloABytes = (kHaloPW * kHaloPH * 128 + 1023) / 1024 * 1024;  // 23552
constexpr int kHaloAStages = 3;   // default number of A patches in flight
constexpr int kMaxAStages = 5;    // weight-stationary layers (ConvParams::wstat) spend the freed B ring on deeper A prefetch
constexpr int kPairAStages = 2;   // pair tile: one patch pair feeds 9 k-blocks, so two pairs in flight suffice
// work-list pair tile: one (8+2)x(8+2)-pixel patch per 8x8 tile, 1024-byte aligned like the halo patch
constexpr int kListPW = kListTile + 2;
static_assert(kListPW == kHaloPW, "the list patches share the halo descriptors' row-group stride");
constexpr int kListABytes = (kListPW * kListPW * 128 + 1023) / 1024 * 1024;  // 13312
constexpr int kBarBytes = 512;
constexpr int kSbBytes = 2 * 2 * 256 * 4;  // per consumer warpgroup: staged (scale, bias) of its current (segment, n-block)
// generic variant: the eSE pool partials handed from warpgroup 1 (rows 0..63) to warpgroup 2 (rows 64..127), per staging
// buffer parity: 128 threads x 8 fp32
constexpr int kPoolXBytes = 2 * 128 * 8 * 4;
constexpr int kMaxStagger = 6;  // k-blocks by which consumer warpgroup 1 leads warpgroup 2 (ConvParams::stagger)
constexpr int kConsumerWarps = 8;

struct TileCoord {
    int seg, img, y0, x0, n_blk;
};

// x / d for 0 <= x < 2^24 without the ~40-instruction integer division: fp32 reciprocal estimate, corrected by one.
__device__ __forceinline__ int fast_div(int x, int d, float inv_d) {
    int q = __float2int_rz(__int2float_rz(x) * inv_d);
    const int r = x - q * d;
    q += (r >= d) ? 1 : 0;
    q -= (r < 0) ? 1 : 0;
    return q;
}

// work item = (M-tile, n-block), n-block fastest.  PAIR: the M unit is a pair of tiles, `sub` selects tile 2i + sub; with
// LIST four 8x8 tiles, `sub` selects 8x8 tile 4i + sub of the list (half `sub & 1` of entry 2i + sub / 2 for 16-row tiles).
// Called by whole warps (the list entry is broadcast from lane 0, so the coordinates stay provably warp-uniform).
template <bool PAIR = false, bool LIST = false>
__device__ __forceinline__ TileCoord decode_tile(const ConvParams& p, int work, int sub = 0) {
    TileCoord t;
    int mt = work;
    t.n_blk = 0;
    if (p.n_blocks > 1) {
        mt = fast_div(work, p.n_blocks, p.inv_n_blocks);
        t.n_blk = work - mt * p.n_blocks;
    }
    int r, half = 0;
    if (LIST) {
        int q = mt;
        if (PAIR) {
            const int sh = p.seg[0].th >> 4;  // 8x8 tiles per entry: 1 (th 8) or 2 (th 16)
            q = (4 * mt + sub) >> sh;
            half = (4 * mt + sub) & sh;
        }
        const uint32_t e = __shfl_sync(0xffffffffu, __ldg(p.tile_list + q), 0);
        t.seg = static_cast<int>(e >> 29);
        t.img = static_cast<int>((e >> 16) & (kTileListMaxImages - 1));
        r = static_cast<int>(e & (kTileListMaxTiles - 1));
    } else {
        int s = 0;
#pragma unroll
        for (int i = 1; i < kMaxSeg; ++i) {
            if (i < p.nseg && mt >= p.seg[i].tile_begin) s = i;
        }
        t.seg = s;
        const ConvSeg& g = p.seg[s];
        int local = mt - g.tile_begin;
        int per_img = g.tiles_x * g.tiles_y;
        if (PAIR) per_img = (per_img + 1) >> 1;
        t.img = fast_div(local, per_img, g.inv_per_img);
        r = local - t.img * per_img;
        if (PAIR) r = 2 * r + sub;
    }
    const ConvSeg& g = p.seg[t.seg];
    int ty = fast_div(r, g.tiles_x, g.inv_tiles_x);
    int tx = r - ty * g.tiles_x;
    t.y0 = ty * g.th + (LIST && PAIR ? kListTile * half : 0);
    t.x0 = tx * g.tw;
    return t;
}

// (a, b) -> packed 16-bit pair; MODE bit 0: ReLU fused into the conversion (cvt.rn.relu), bit 1: fp16 instead of bf16.
template <int MODE>
__device__ __forceinline__ uint32_t pack2_mode(float a, float b) {
    uint32_t r;
    if (MODE == 0) {
        asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
    } else if (MODE == 1) {
        asm("cvt.rn.relu.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
    } else if (MODE == 2) {
        asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
    } else {
        asm("cvt.rn.relu.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
    }
    return r;
}

template <bool F16>
__device__ __forceinline__ uint32_t pack2_relu(float a, float b, bool relu) {
    return relu ? pack2_mode<(F16 ? 2 : 0) | 1>(a, b) : pack2_mode<F16 ? 2 : 0>(a, b);
}

// elect.sync: exactly one lane of the (converged) warp gets true.  Keeping the producer loops warp-converged and
// predicating only the issue instructions on the elected lane lets the compiler keep the TMA operands in uniform registers.
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile(
        "{\n\t.reg .b32 rx;\n\t.reg .pred px;\n\t"
        "elect.sync rx|px, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, px;\n\t}"
        : "=r"(pred));
    return pred != 0;
}

// One warpgroup's wgmmas of one k-block: four K = 16 steps, one commit group.  Channels beyond cin are zero in both operands
// (TMA zero-fills the activation channels past C, the packed weights are zero there), so the padded steps add exact zeros;
// issuing them unconditionally keeps the wgmma chain free of control flow, which ptxas would otherwise serialize.
template <int N, bool F16, int L>
__device__ __forceinline__ void mma_kblock(float (&acc)[L], uint64_t adesc, uint64_t bdesc, bool first) {
    wg::fence();
#pragma unroll
    for (int k = 0; k < kBlockK / 16; ++k) wg::wgmma<N, F16>(acc, adesc + 2 * k, bdesc + 2 * k, (first && k == 0) ? 0u : 1u);
    wg::commit();
}

// Pair tile: the same k-block for both 64-row halves of the warpgroup's sub-tile (one B descriptor, two A descriptors).
template <int N, bool F16, int L>
__device__ __forceinline__ void mma_kblock2(float (&acc0)[L], float (&acc1)[L], uint64_t adesc0, uint64_t adesc1,
                                            uint64_t bdesc, bool first) {
    wg::fence();
#pragma unroll
    for (int k = 0; k < kBlockK / 16; ++k) {
        const uint32_t scale_d = (first && k == 0) ? 0u : 1u;
        wg::wgmma<N, F16>(acc0, adesc0 + 2 * k, bdesc + 2 * k, scale_d);
        wg::wgmma<N, F16>(acc1, adesc1 + 2 * k, bdesc + 2 * k, scale_d);
    }
    wg::commit();
}

// BN = block_n, the wgmma N: a compile-time parameter, so the accumulators are exactly BN / 2 registers per consumer thread
// and 64-row half (PAIR: two halves per warpgroup)
template <bool HALO, bool F16, int BN, bool PAIR = false, bool LIST = false>
__global__ void __launch_bounds__(kConvThreads, 1) conv_igemm_kernel(const __grid_constant__ ConvParams p) {
    static_assert(!PAIR || (HALO && BN == 128), "the pair tile is a halo variant with block_n 128");
    static_assert(!LIST || PAIR, "work-list mode is instantiated for the pair tile only");
    constexpr int MH = PAIR ? 2 : 1;                                   // 64-row halves per consumer warpgroup
    // one A stage: the patch of every sub-tile (LIST: of every 8x8 tile)
    constexpr int kASlot = LIST ? 4 * kListABytes : PAIR ? 2 * kHaloABytes : kHaloABytes;
    extern __shared__ uint8_t smem_raw[];
    // 128B-swizzled tiles need 1024-byte alignment
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    // generic: num_stages x [A 16 KiB | B block_n*128].  halo: num_stages x [B block_n*128], then a_stages x [A patch 23 KiB
    // (PAIR: two patches; LIST: four 13 KiB patches)], then the staging tiles (PAIR: two per consumer warpgroup)
    const int stage_bytes = (HALO ? 0 : kABytes) + BN * 128;
    // weight-stationary (HALO, one n-block, cin <= 64): ALL k-blocks of the weight tensor stay resident in the B region
    // (loaded once per CTA) instead of cycling through the stage ring for every tile
    const bool wstat = HALO && !PAIR && p.wstat != 0;
    const int a_stages = HALO ? p.a_stages : 0;
    uint8_t* halo_a = smem + (wstat ? p.taps * p.kchunks : p.num_stages) * stage_bytes;
    uint8_t* staging = halo_a + a_stages * kASlot;
    uint64_t* bars = reinterpret_cast<uint64_t*>(staging + 2 * MH * kStagingBytes);
    uint64_t* full_bar = bars;                     // [kMaxStages]
    uint64_t* empty_bar = bars + kMaxStages;       // [kMaxStages]
    uint64_t* afull_bar = bars + 2 * kMaxStages;   // [kMaxAStages]
    uint64_t* aempty_bar = afull_bar + kMaxAStages;
    uint64_t* wfull_bar = aempty_bar + kMaxAStages;  // [1] resident weights landed (wstat)
    uint64_t* skew_bar = wfull_bar + 1;              // [1] warpgroup 1 has issued p.stagger k-blocks of its first item
    uint64_t* poolx_full = skew_bar + 1;             // [2] eSE partials of rows 0..63 handed over (per staging parity)
    uint64_t* poolx_empty = poolx_full + 2;          // [2] ... and taken
    // shared-window addresses of the epilogue's staging tiles, the staged folded-BN vectors (per consumer warpgroup) and
    // the eSE partials hand-over (explicit LDS / STS)
    const uint32_t staging_u32 = ptx::smem_u32(staging);
    const uint32_t sb_u32 = ptx::smem_u32(reinterpret_cast<uint8_t*>(bars) + kBarBytes);
    const uint32_t poolx_u32 = sb_u32 + kSbBytes;

    const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);  // provably warp-uniform
    const int lane = threadIdx.x & 31;

    if (warp == 0 && lane == 0) {
        ptx::prefetch_tensormap(&p.w_map);
        for (int s = 0; s < p.nseg; ++s) {
            ptx::prefetch_tensormap(&p.seg[s].in_map[0]);
            if (p.out_mode == 0) ptx::prefetch_tensormap(&p.seg[s].out_map);
        }
        for (int i = 0; i < p.num_stages; ++i) {
            ptx::mbar_init(&full_bar[i], HALO ? 1 : 2);  // generic: A (warp 0) + B (warp 2) each arrive.expect_tx
            ptx::mbar_init(&empty_bar[i], kConsumerWarps);
        }
        for (int i = 0; i < kMaxAStages; ++i) {
            ptx::mbar_init(&afull_bar[i], 1);
            ptx::mbar_init(&aempty_bar[i], kConsumerWarps);
        }
        ptx::mbar_init(wfull_bar, 1);
        ptx::mbar_init(skew_bar, 1);
        for (int i = 0; i < 2; ++i) {
            ptx::mbar_init(&poolx_full[i], 128);
            ptx::mbar_init(&poolx_empty[i], 128);
        }
        ptx::fence_barrier_init();
    }
    __syncthreads();
    // Programmatic dependent launch: everything above (barrier init, descriptor prefetch) overlapped the tail of the
    // previous kernel in the stream; from here on we touch its outputs, so wait for it, and let the next kernel start its
    // own prologue as our CTAs retire.
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

    const int kblocks = p.taps * p.kchunks;
    const int w_first = static_cast<int>(blockIdx.x), w_step = static_cast<int>(gridDim.x);
    int w_total = p.total_work;
    if (LIST) {  // work-list mode: the list was written by an earlier kernel of the stream
        const int units = PAIR ? ((__ldg(p.tile_count) << (p.seg[0].th >> 4)) >> 2) : __ldg(p.tile_count);
        w_total = __shfl_sync(0xffffffffu, units, 0) * p.n_blocks;
    }

    if (warp == 0) {
        // ---------------------------------------------------------------- warp 0: activation (A) producer in the
        // generic variant, weight (B) producer in the halo variant.  Whole warp runs the loop; one elected lane issues.
        int stage = 0;
        uint32_t phase = 0;
        if (wstat) {
            // the whole weight tensor (<= 9 x 8 KiB), once: one barrier, one transaction count
            if (elect_one()) {
                ptx::mbar_expect_tx(wfull_bar, kblocks * p.block_n * 128);
                for (int kb = 0; kb < kblocks; ++kb)
                    ptx::tma_load_2d(smem + kb * stage_bytes, &p.w_map, wfull_bar, kb * kBlockK, 0);
            }
            __syncwarp();
        }
        for (int work = w_first; work < w_total && !wstat; work += w_step) {
            const TileCoord t = decode_tile<PAIR, LIST>(p, work);
            const ConvSeg& g = p.seg[t.seg];
            if (HALO) {
                for (int kc = 0; kc < p.kchunks; ++kc) {
                    for (int tap = 0; tap < 9; ++tap) {
                        ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
                        if (elect_one()) {
                            ptx::mbar_expect_tx(&full_bar[stage], p.block_n * 128);
                            ptx::tma_load_2d(smem + stage * stage_bytes, &p.w_map, &full_bar[stage],
                                             (tap * p.kchunks + kc) * kBlockK, t.n_blk * p.block_n);
                        }
                        __syncwarp();
                        if (++stage == p.num_stages) {
                            stage = 0;
                            phase ^= 1;
                        }
                    }
                }
                continue;
            }
            const int a_c0 = p.grouped ? t.n_blk * kBlockK : 0;  // block-diagonal: n-block j reads channels 64 j..
            for (int tap = 0; tap < p.taps; ++tap) {
                const int r = (p.taps == 9) ? tap / 3 : 1;
                const int s = (p.taps == 9) ? tap - 3 * (tap / 3) : 1;
                for (int kc = 0; kc < p.kchunks; ++kc) {
                    ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
                    if (elect_one()) {
                        uint8_t* a_dst = smem + stage * stage_bytes;
                        ptx::mbar_expect_tx(&full_bar[stage], kABytes);  // the weight tile is armed + issued by warp 2
                        if (p.stride == 1) {
                            ptx::tma_load_4d(a_dst, &g.in_map[0], &full_bar[stage], a_c0 + kc * kBlockK, t.x0 + s - 1,
                                             t.y0 + r - 1, t.img);
                        } else {
                            // stride 2: input (2*oy + r - 1, 2*ox + s - 1) in the parity-split view [B][H/2][2][W/2][wp*C..]
                            const int wp = (s == 1) ? 0 : 1;
                            const int dw = (s == 0) ? -1 : 0;
                            const int hp = (r == 1) ? 0 : 1;
                            const int dh = (r == 0) ? -1 : 0;
                            ptx::tma_load_5d(a_dst, &g.in_map[wp], &full_bar[stage], a_c0 + kc * kBlockK, t.x0 + dw, hp,
                                             t.y0 + dh, t.img);
                        }
                    }
                    __syncwarp();
                    if (++stage == p.num_stages) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
            }
        }
    } else if (warp == 2) {
        if (!HALO) {
            // ------------------------------------------------------------ warp 2: weight-tile (B) producer (generic)
            int stage = 0;
            uint32_t phase = 0;
            const uint32_t b_bytes = p.block_n * 128;
            for (int work = w_first; work < w_total; work += w_step) {
                const int n0 = (work % p.n_blocks) * p.block_n;
                for (int kb = 0; kb < kblocks; ++kb) {
                    ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
                    if (elect_one()) {
                        ptx::mbar_expect_tx(&full_bar[stage], b_bytes);
                        ptx::tma_load_2d(smem + stage * stage_bytes + kABytes, &p.w_map, &full_bar[stage], kb * kBlockK, n0);
                    }
                    __syncwarp();
                    if (++stage == p.num_stages) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
            }
        } else {
            // ------------------------------------------------------------ warp 2: halo A-patch producer: one box
            // [18][10][64 ch] (180 rows of 128 B, 128B-swizzled, zero-filled outside the image) per 64-channel block
            // (PAIR: one per sub-tile, both on one barrier; LIST: one [10][10] box per 8x8 tile, all four on one barrier)
            int as = 0;
            uint32_t aphase = 0;
            for (int work = w_first; work < w_total; work += w_step) {
                const TileCoord t = decode_tile<PAIR, LIST>(p, work);
                const TileCoord t1 = PAIR ? decode_tile<PAIR, LIST>(p, work, 1) : t;
                const ConvSeg& g = p.seg[t.seg];
                const int a_c0 = p.grouped ? t.n_blk * kBlockK : 0;  // block-diagonal: n-block j reads channels 64 j..
                // LIST: four [10][10] patches, one per listed 8x8 tile
                const TileCoord t2 = LIST ? decode_tile<PAIR, LIST>(p, work, 2) : t;
                const TileCoord t3 = LIST ? decode_tile<PAIR, LIST>(p, work, 3) : t;
                constexpr int a_bytes = LIST ? 4 * kListPW * kListPW * 128 : MH * kHaloPW * kHaloPH * 128;
                constexpr int patch = LIST ? kListABytes : kHaloABytes;  // patch spacing in the A stage
                for (int kc = 0; kc < p.kchunks; ++kc) {
                    ptx::mbar_wait(&aempty_bar[as], aphase ^ 1);
                    if (elect_one()) {
                        ptx::mbar_expect_tx(&afull_bar[as], a_bytes);
                        ptx::tma_load_4d(halo_a + as * kASlot, &g.in_map[0], &afull_bar[as], a_c0 + kc * kBlockK, t.x0 - 1,
                                         t.y0 - 1, t.img);
                        if (PAIR)
                            ptx::tma_load_4d(halo_a + as * kASlot + patch, &g.in_map[0], &afull_bar[as], kc * kBlockK,
                                             t1.x0 - 1, t1.y0 - 1, t1.img);
                        if (LIST) {
                            ptx::tma_load_4d(halo_a + as * kASlot + 2 * patch, &g.in_map[0], &afull_bar[as], kc * kBlockK,
                                             t2.x0 - 1, t2.y0 - 1, t2.img);
                            ptx::tma_load_4d(halo_a + as * kASlot + 3 * patch, &g.in_map[0], &afull_bar[as], kc * kBlockK,
                                             t3.x0 - 1, t3.y0 - 1, t3.img);
                        }
                    }
                    __syncwarp();
                    if (++as == a_stages) {
                        as = 0;
                        aphase ^= 1;
                    }
                }
            }
        }
    } else if (warp >= 4) {
        // ---------------------------------------------------------------- consumer warpgroups 1, 2
        // Each warpgroup runs its epilogue on its own: its own staging buffers, named barrier, store leader and copy of the
        // folded-BN vectors, so neither waits for the other between work items.  Warpgroup 2 starts p.stagger k-blocks
        // behind warpgroup 1; the shared ring then keeps them staggered (DESIGN.md section 3): one warpgroup's epilogue
        // runs while the other one's wgmmas keep the tensor pipe busy.
        const int wgi = (warp >> 2) - 1;                                 // rows 64 * wgi .. (PAIR: sub-tile wgi)
        const int wt = static_cast<int>(threadIdx.x) & 127;              // thread of the warpgroup
        const int wl = warp & 3;
        const bool store_leader = wt == 0;
        const uint32_t epi_bar = 2 + wgi;
        const uint32_t s_scale_u32 = sb_u32 + wgi * (kSbBytes / 2);  // [256] fp32 scale
        const uint32_t s_bias_u32 = s_scale_u32 + 256 * 4;           // [256] fp32 bias
        const int out_mode = PAIR ? 0 : p.out_mode;
        const uint64_t desc_hi = ptx::make_sw128_desc(0, HALO ? kHaloPW * 128 : 1024) & ~0x3FFFull;
        const uint64_t bdesc_hi = ptx::make_sw128_desc(0, 1024) & ~0x3FFFull;
        const uint32_t smem_lo = ptx::smem_u32(smem) >> 4;
        const uint32_t halo_lo = ptx::smem_u32(halo_a) >> 4;
        const uint32_t stage_units = static_cast<uint32_t>(stage_bytes) >> 4;
        // the rows of this thread's accumulator row-halves within the warpgroup's staging tile (2 per 64-row half); row0 + row
        // is the pixel within the 128-pixel tile
        const int row0 = PAIR ? 0 : 64 * wgi;
        int row[2 * MH];
#pragma unroll
        for (int m = 0; m < MH; ++m) {
            row[2 * m] = 64 * m + 16 * wl + (lane >> 2);
            row[2 * m + 1] = row[2 * m] + 8;
        }
        const int qc = 2 * (lane & 3);  // first of this thread's two columns in every 8-column group
        float acc[MH][BN / 2];
        int stage = 0;
        uint32_t phase = 0;
        int as = 0;
        uint32_t aphase = 0;
        int sbuf = 0;
        uint32_t poolx_phase = 0;  // bit b: phase of the eSE hand-over of staging parity b
        int sb_key = -1;  // (segment, n-block) whose folded-BN vectors are staged in s_scale / s_bias
        if (wstat) ptx::mbar_wait(wfull_bar, 0);
        if (wgi == 1 && p.stagger > 0 && w_first < w_total) ptx::mbar_wait(skew_bar, 0);
        // warpgroup 1 releases warpgroup 2 once it has issued k-block p.stagger - 1 (<= kblocks - 1) of its first item
        bool skew_pending = wgi == 0 && wt == 0 && p.stagger > 0;
        auto skew_arrive = [&](int i) {
            if (skew_pending && i + 1 == p.stagger) {
                ptx::mbar_arrive(skew_bar);
                skew_pending = false;
            }
        };
        for (int work = w_first; work < w_total; work += w_step) {
            const TileCoord t = decode_tile<PAIR, LIST>(p, work, LIST ? 2 * wgi : PAIR ? wgi : 0);
            const ConvSeg& g = p.seg[t.seg];
            // ---- main loop: one commit group per k-block; the slot (and halo patch) of group i is released after
            // group i + 1 has been issued and group i has retired (wait_group 1)
            int rel_stage = -1, rel_as = -1;
            auto release = [&]() {
                if (lane == 0) {
                    if (rel_stage >= 0) ptx::mbar_arrive(&empty_bar[rel_stage]);
                    if (rel_as >= 0) ptx::mbar_arrive(&aempty_bar[rel_as]);
                }
                rel_stage = -1;
                rel_as = -1;
            };
            if (HALO) {
                for (int kc = 0; kc < p.kchunks; ++kc) {
                    ptx::mbar_wait(&afull_bar[as], aphase);
                    // rows 64 * wgi.. of the tile's patch; PAIR: row 0 of sub-tile wgi's patch (rows 64.. are 8 patch rows on);
                    // LIST: row 0 of 8x8 tile 2 wgi's patch (rows 64.. are those of tile 2 wgi + 1, the next patch)
                    const uint32_t a_lo = halo_lo + static_cast<uint32_t>(as) * (kASlot >> 4) +
                                          (LIST   ? 2 * wgi * (kListABytes >> 4)
                                           : PAIR ? wgi * (kHaloABytes >> 4)
                                                  : wgi * 8 * kHaloPW * 8);
                    constexpr uint32_t half1 = LIST ? kListABytes >> 4 : 8 * kHaloPW * 8;  // rows 64.. (PAIR)
                    for (int tap = 0; tap < 9; ++tap) {
                        if (!wstat) ptx::mbar_wait(&full_bar[stage], phase);
                        const int r = tap / 3, s = tap - 3 * r;
                        const uint32_t a_tap = a_lo + (r * kHaloPW + s) * 8;  // whole pixels: 128 B = 8 x 16 B
                        const uint32_t b_lo =
                            smem_lo + static_cast<uint32_t>(wstat ? tap * p.kchunks + kc : stage) * stage_units;
                        if constexpr (PAIR)
                            mma_kblock2<BN, F16>(acc[0], acc[MH - 1], desc_hi | a_tap, desc_hi | (a_tap + half1),
                                                 bdesc_hi | b_lo, (kc | tap) == 0);
                        else
                            mma_kblock<BN, F16>(acc[0], desc_hi | a_tap, bdesc_hi | b_lo, (kc | tap) == 0);
                        skew_arrive(9 * kc + tap);
                        wg::wait<1>();
                        release();
                        rel_stage = wstat ? -1 : stage;
                        if (tap == 8) rel_as = as;
                        if (!wstat && ++stage == p.num_stages) {
                            stage = 0;
                            phase ^= 1;
                        }
                    }
                    if (++as == a_stages) {
                        as = 0;
                        aphase ^= 1;
                    }
                }
            } else {
                for (int kb = 0; kb < kblocks; ++kb) {
                    ptx::mbar_wait(&full_bar[stage], phase);
                    const uint32_t a_lo = smem_lo + static_cast<uint32_t>(stage) * stage_units + wgi * (64 * 128 / 16);
                    const uint32_t b_lo = smem_lo + static_cast<uint32_t>(stage) * stage_units + (kABytes >> 4);
                    mma_kblock<BN, F16>(acc[0], desc_hi | a_lo, bdesc_hi | b_lo, kb == 0);
                    skew_arrive(kb);
                    wg::wait<1>();
                    release();
                    rel_stage = stage;
                    if (++stage == p.num_stages) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
            }
            wg::wait<0>();
            release();
#pragma unroll
            for (int m = 0; m < MH; ++m) wg::fence_regs(acc[m]);

            // ---- epilogue of this warpgroup's 64 rows (PAIR: of its 128-row sub-tile)
            const int n_base = t.n_blk * BN;
            const int tw = HALO ? kHaloTw : g.tw, tw_shift = HALO ? 3 : g.tw_shift;  // the halo tile is 16 x 8
            static_assert(kHaloTw == 8 && kListTile == 8, "tw_shift of the halo and list tiles");
            // origin of each 64-row half in the frame of rows (row0 + row) >> tw_shift.  LIST: half 1 is the warpgroup's second
            // 8x8 tile, whose rows 64.. sit 8 tile rows below that origin
            int y_org[MH], x_org[MH];
#pragma unroll
            for (int m = 0; m < MH; ++m) {
                y_org[m] = t.y0;
                x_org[m] = t.x0;
            }
            if constexpr (LIST) {
                const TileCoord t1 = decode_tile<PAIR, LIST>(p, work, 2 * wgi + 1);
                y_org[1] = t1.y0 - kListTile;
                x_org[1] = t1.x0;
            }
            bool in_img[2 * MH];
            const __nv_bfloat16* res_ptr[2 * MH];
            float* f32_ptr[2 * MH];
#pragma unroll
            for (int h = 0; h < 2 * MH; ++h) {
                const int ly = (row0 + row[h]) >> tw_shift;
                const int lx = (row0 + row[h]) - (ly << tw_shift);
                const int oy = y_org[h >> 1] + ly, ox = x_org[h >> 1] + lx;
                in_img[h] = (oy < g.H) && (ox < g.W);
                res_ptr[h] = nullptr;
                if (g.residual != nullptr && in_img[h]) {
                    const int ry = g.res_up2 ? (oy >> 1) : oy;
                    const int rx = g.res_up2 ? (ox >> 1) : ox;
                    res_ptr[h] =
                        g.residual + (static_cast<size_t>(t.img * g.res_H + ry) * g.res_W + rx) * g.res_pitch + n_base + qc;
                }
                f32_ptr[h] = nullptr;
                if (out_mode == 1 && in_img[h])
                    f32_ptr[h] = g.out_f32 + (static_cast<size_t>(t.img * g.H + oy) * g.W + ox) * g.out_pitch + n_base + qc;
            }
            // per-channel (scale, bias) of this (segment, n-block) in this warpgroup's shared copy: broadcast LDS instead of LDG
            // with their 64-bit address arithmetic.  The first barrier waits for the warpgroup's readers of the previous copy.
            const int key = t.seg * 64 + t.n_blk;
            if (key != sb_key) {
                ptx::named_bar_sync(epi_bar, 128);
                sb_key = key;
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int ch = wt + 128 * i;
                    if (ch < BN) {
                        ptx::st_shared_f32(s_scale_u32 + ch * 4, __ldg(g.scale + n_base + ch));
                        ptx::st_shared_f32(s_bias_u32 + ch * 4, __ldg(g.bias + n_base + ch));
                    }
                }
                ptx::named_bar_sync(epi_bar, 128);
            }
            const bool has_res = g.residual != nullptr;

#pragma unroll
            for (int c = 0; c < (BN + 63) / 64; ++c) {
                const int c0 = 64 * c;
                // this warpgroup's staging buffer of parity sbuf: MH x 64 rows
                const int sb_off = (2 * wgi + sbuf) * MH * kHalfStagingBytes;
                uint8_t* stag = staging + sb_off;
                const uint32_t stag_u32 = staging_u32 + sb_off;
                if (out_mode == 0) {
                    // the TMA store that last read this staging buffer must have drained
                    if (store_leader) ptx::tma_store_wait_read<1>();
                    ptx::named_bar_sync(epi_bar, 128);
                }
#pragma unroll
                for (int jj = 0; jj < 8; ++jj) {
                    const int j = 8 * c + jj;  // 8-column group of the tile
                    if (8 * j >= BN) break;
                    const int col = 8 * j + qc;
                    const float2 sc = ptx::ld_shared_f2(s_scale_u32 + col * 4);
                    const float2 bi = ptx::ld_shared_f2(s_bias_u32 + col * 4);
#pragma unroll
                    for (int h = 0; h < 2 * MH; ++h) {
                        float y0 = fmaf(acc[h >> 1][4 * j + 2 * (h & 1)], sc.x, bi.x);
                        float y1 = fmaf(acc[h >> 1][4 * j + 2 * (h & 1) + 1], sc.y, bi.y);
                        if (has_res) {
                            const uint32_t rv =
                                res_ptr[h] != nullptr ? __ldg(reinterpret_cast<const unsigned int*>(res_ptr[h] + 8 * j)) : 0u;
                            const float2 f = F16 ? unpack2_f16(rv) : unpack2_bf16(rv);
                            y0 += f.x;
                            y1 += f.y;
                        }
                        if (out_mode == 0) {
                            const int r = row[h];
                            ptx::st_shared_u32(stag_u32 + r * 128 + ((jj ^ (r & 7)) << 4) + qc * 2,
                                               pack2_relu<F16>(y0, y1, p.relu != 0));
                        } else if (f32_ptr[h] != nullptr) {
                            if (p.relu) {
                                y0 = fmaxf(y0, 0.0f);
                                y1 = fmaxf(y1, 0.0f);
                            }
                            if (g.lo != nullptr) {
                                const float2 lo = __ldg(reinterpret_cast<const float2*>(g.lo + n_base + col));
                                y0 = fmaxf(y0, lo.x);
                                y1 = fmaxf(y1, lo.y);
                            }
                            *reinterpret_cast<float2*>(f32_ptr[h] + 8 * j) = make_float2(y0, y1);
                        }
                    }
                }
                if (out_mode == 0) {
                    ptx::fence_proxy_async_smem();  // generic-proxy smem writes -> visible to the TMA engine
                    ptx::named_bar_sync(epi_bar, 128);
                    if (store_leader) {
                        // one box per 64-pixel half: the out map's box is the first 64 pixels of a tile in row-major order
#pragma unroll
                        for (int m = 0; m < MH; ++m) {
                            const int px = 64 * (PAIR ? m : wgi);
                            ptx::tma_store_4d(&g.out_map, stag + m * kHalfStagingBytes, n_base + c0, x_org[m] + (px & (tw - 1)),
                                              y_org[m] + (px >> tw_shift), t.img);
                        }
                        ptx::tma_store_commit();
                    }
                    if (!HALO && !PAIR && g.pool_partial != nullptr) {
                        // eSE global-average-pool, fused: per-tile channel sums of the 16-bit tile just staged (exactly the
                        // values the reference pools, vovnet.py:181).  Thread e covers channels 8*(e&7).. of rows
                        // (e>>3) + 16*i; the 4 row-groups of a warp are shuffle-reduced; one fp32 partial per
                        // (tile, warp, channel) -> deterministic reduction later (no atomics).  Rows i < 4 are warpgroup 1's:
                        // thread e of warpgroup 1 hands its running sums to thread e of warpgroup 2, which adds rows i >= 4 in
                        // the same order, reduces and stores.
                        const int e = wt;
                        const int cg = e & 7;
                        const uint32_t px_u32 = poolx_u32 + sbuf * (kPoolXBytes / 2) + e * 16;
                        const uint32_t par = (poolx_phase >> sbuf) & 1;
                        float ps[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
                        if (wgi == 1) {
                            ptx::mbar_wait(&poolx_full[sbuf], par);
                            const float4 a = ptx::ld_shared_f4(px_u32), b = ptx::ld_shared_f4(px_u32 + 128 * 16);
                            ps[0] = a.x, ps[1] = a.y, ps[2] = a.z, ps[3] = a.w;
                            ps[4] = b.x, ps[5] = b.y, ps[6] = b.z, ps[7] = b.w;
                            ptx::mbar_arrive(&poolx_empty[sbuf]);
                        }
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const int r = (e >> 3) + 16 * i;  // row of the staging buffer, row0 + r of the tile
                            const int ry = t.y0 + ((row0 + r) >> g.tw_shift), rx = t.x0 + ((row0 + r) & (g.tw - 1));
                            if (ry < g.H && rx < g.W) {
                                const uint4 u = ptx::ld_shared_v4(stag_u32 + r * 128 + ((cg ^ (r & 7)) << 4));
                                const uint32_t* b2 = reinterpret_cast<const uint32_t*>(&u);
#pragma unroll
                                for (int j = 0; j < 4; ++j) {
                                    const float2 f = unpack2_act(b2[j], F16 ? 1 : 0);
                                    ps[2 * j] += f.x;
                                    ps[2 * j + 1] += f.y;
                                }
                            }
                        }
                        if (wgi == 0) {
                            ptx::mbar_wait(&poolx_empty[sbuf], par ^ 1);
                            ptx::st_shared_f4(px_u32, make_float4(ps[0], ps[1], ps[2], ps[3]));
                            ptx::st_shared_f4(px_u32 + 128 * 16, make_float4(ps[4], ps[5], ps[6], ps[7]));
                            ptx::mbar_arrive(&poolx_full[sbuf]);
                        }
                        poolx_phase ^= 1u << sbuf;
                        if (wgi == 1) {
#pragma unroll
                            for (int j = 0; j < 8; ++j) {
                                ps[j] += __shfl_xor_sync(0xffffffffu, ps[j], 8);
                                ps[j] += __shfl_xor_sync(0xffffffffu, ps[j], 16);
                            }
                            if (lane < 8 && c0 + cg * 8 < BN) {
                                const int tile_in_img = (t.y0 / g.th) * g.tiles_x + (t.x0 / g.tw);
                                float* dst = g.pool_partial +
                                             ((static_cast<size_t>(t.img) * (g.tiles_x * g.tiles_y) + tile_in_img) * 4 + (e >> 5)) *
                                                 g.pool_pitch +
                                             n_base + c0 + cg * 8;
                                *reinterpret_cast<float4*>(dst) = make_float4(ps[0], ps[1], ps[2], ps[3]);
                                *reinterpret_cast<float4*>(dst + 4) = make_float4(ps[4], ps[5], ps[6], ps[7]);
                            }
                        }
                    }
                    sbuf ^= 1;
                }
            }
        }
        if (store_leader) ptx::tma_store_wait_all();
    }
}

}  // namespace

// Kernel of one (halo, fp16, block_n) combination, or nullptr when block_n is not in this translation unit's group.
using ConvKernel = void (*)(ConvParams);
#define DD3D_CONV_KERNEL_CASE(N)                                                                                         \
    case N:                                                                                                              \
        return halo ? (fp16 ? conv_igemm_kernel<true, true, N> : conv_igemm_kernel<true, false, N>)                     \
                    : (fp16 ? conv_igemm_kernel<false, true, N> : conv_igemm_kernel<false, false, N>);
#define DD3D_CONV_KERNEL_GROUP(NAME, N0, N1, N2, N3)                                                                     \
    ConvKernel NAME(bool halo, bool fp16, int block_n) {                                                                 \
        switch (block_n) {                                                                                               \
            DD3D_CONV_KERNEL_CASE(N0)                                                                                    \
            DD3D_CONV_KERNEL_CASE(N1)                                                                                    \
            DD3D_CONV_KERNEL_CASE(N2)                                                                                    \
            DD3D_CONV_KERNEL_CASE(N3)                                                                                    \
            default: return nullptr;                                                                                     \
        }                                                                                                                \
    }
ConvKernel conv_kernel_n16_64(bool halo, bool fp16, int block_n);
ConvKernel conv_kernel_n80_128(bool halo, bool fp16, int block_n);
ConvKernel conv_kernel_pair(bool fp16, bool list);  // the pair-tile halo kernel (block_n 128), in conv_igemm_n80_128.cu
ConvKernel conv_kernel_n144_192(bool halo, bool fp16, int block_n);
ConvKernel conv_kernel_n208_256(bool halo, bool fp16, int block_n);

}  // namespace dd3d
