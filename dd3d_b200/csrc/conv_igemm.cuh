// Implicit-GEMM convolution on Hopper tensor cores (sm_90a, wgmma): interface.
//
// One launch covers up to kMaxSeg "segments" (FPN levels) that share one weight tensor (the FCOS towers share
// weights across levels, reference fcos2d.py:74-91 / fcos3d.py:81-100) but have their own activation tensors,
// spatial sizes and folded-BN epilogue vectors (ModuleListDial, normalization.py:30-40).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace dd3d {

constexpr int kMaxSeg = 5;
constexpr int kBlockM = 128;  // output pixels per tile (th * tw)
constexpr int kBlockK = 64;   // bf16 channels per k-block = one 128-byte swizzle row
constexpr int kConvThreads = 384;  // warpgroup 0: TMA producers (warps 0, 2); warpgroups 1, 2: wgmma + epilogue, 64 rows each

struct ConvSeg {
    CUtensorMap in_map[2];  // NHWC bf16 input.  stride 1: [0] (4-D).  stride 2: [w-parity] (5-D parity split)
    CUtensorMap out_map;    // NHWC bf16 output (out_mode 0), 4-D, TMA store clips partial tiles
    const float* scale;     // [n_pad] folded BN scale (1 when no norm)
    const float* bias;      // [n_pad] folded BN bias / conv bias
    const float* lo;        // [n_pad] per-channel lower clamp (out_mode 1 only; -inf = none) or nullptr
    const __nv_bfloat16* residual;  // NHWC bf16 added before the activation, or nullptr
    float* out_f32;         // out_mode 1: NHWC fp32, pitch out_pitch
    int res_pitch, res_up2, res_H, res_W;  // res_up2: residual is the 2x-coarser map (FPN nearest upsample)
    int out_pitch;
    int H, W;         // OUTPUT spatial size
    int th, tw;       // tile shape, th * tw == 128
    int tiles_x, tiles_y;
    int tile_begin;   // index of this segment's first M-tile
    int tw_shift;     // log2(tw)
    float inv_per_img, inv_tiles_x;  // reciprocals for the division-free tile decode (conv_finalize_params)
    void* out16;          // taps-in-N variant, out_mode 0: NHWC 16-bit output written directly (pitch out_pitch)
    float* pool_partial;  // optional [B][tiles_per_image][4][pool_pitch] per-tile channel sums (eSE avg-pool), or nullptr
    int pool_pitch;
};

struct ConvParams {
    CUtensorMap w_map;  // weights [cout_pad][taps * kchunks * 64] bf16, K contiguous
    ConvSeg seg[kMaxSeg];
    int nseg;
    int B;
    int taps;      // 1 or 9
    int stride;    // 1 or 2 (3x3 only)
    int kchunks;   // ceil(cin / 64)
    int n_blocks;  // cout_pad / block_n
    int block_n;   // wgmma N (multiple of 16, <= 256)
    int relu;
    int out_mode;  // 0: bf16 via TMA store, 1: fp32 direct
    int total_work;  // (sum of M-tiles) * n_blocks
    int num_stages;
    int cin;          // real input channels
    int halo;  // 1: 3x3 stride-1 halo-reuse variant (tile 16x8, A patch loaded once per 64-channel block)
    float inv_n_blocks;
    int taps_n;       // 1: taps-in-N variant for 3x3 stride-1 convs with <= 16 output channels (conv_taps_kernel)
    int fp16;         // 16-bit storage type of activations and weights: 0 bf16, 1 fp16 (act16.cuh)
    int wstat;        // 1: weight-stationary halo variant -- all taps * kchunks weight blocks resident in shared memory
    int a_stages;     // halo variants: A patches in flight (3, or up to 5 with wstat; 2 pairs of patches with pair)
    int pair;         // 1: pair-tile halo variant -- work item = two 16x8 tiles x one 128-channel n-block (conv_select_pair)
    // 1: block-diagonal grouped 3x3 (ResNeXt conv2 with channels per group dividing 64): block_n 64, kchunks 1, and the A
    // operand of n-block j is input channels [64 j, 64 j + 64) -- the only channels its 64 output channels read.  Weights
    // [cout][9][64] hold each row's group at its position in the 64-channel block and zeros elsewhere (exact zeros).
    int grouped;
    // Work-list mode (nullptr: every tile of every segment).  The M units come from the entries of tile_list, each
    // (seg << 29) | (img << 16) | (row-major tile of the image); *tile_count entries, read on the device after
    // griddepcontrol.wait.  total_work then only sizes the grid.  Taps-in-N: one 16x8 tile per entry and unit.  Pair tile:
    // the segments' tiles are kListTile wide and th = kListTile (the sparse towers: entries 4i .. 4i + 3 form unit i) or 16
    // rows high (two 8x8 tiles per entry: entries 2i, 2i + 1 form unit i); the entries of a unit lie in one (segment, image).
    const uint32_t* tile_list;
    const int32_t* tile_count;
    // k-blocks consumer warpgroup 2 starts behind warpgroup 1 (0: both start together); conv_finalize_params picks it so
    // that num_stages >= stagger + 2 and the leading warpgroup keeps TMA lookahead
    int stagger;
};
constexpr int kTileListMaxImages = 1 << 13, kTileListMaxTiles = 1 << 16;  // field widths of a tile_list entry
static_assert(sizeof(ConvParams) <= 4096, "kernel parameter space");

// Host helpers (conv_igemm.cu)
const char* conv_last_error();
bool make_act_map(CUtensorMap* map, const void* base, int B, int H, int W, int C, int pitch, int th, int tw, int fp16 = 0);
bool make_act_map_s2(CUtensorMap* map, const void* base, int wp, int B, int H, int W, int C, int pitch, int th,
                     int tw, int fp16 = 0);
// Output map of the conv kernel (out_mode 0) for tiles tw pixels wide: the box is one consumer warpgroup's half of the
// 128-pixel tile, its first 64 pixels in row-major order (64 / tw rows of tw pixels, or 1 x 64 for the 1 x 128 tile).
bool make_out_map(CUtensorMap* map, const void* base, int B, int H, int W, int C, int pitch, int tw, int fp16 = 0);
bool make_weight_map(CUtensorMap* map, const void* base, int ktot, int cout_pad, int block_n, int fp16 = 0);
void choose_tile(int H, int W, int* th, int* tw);
int conv_tiles_per_image(int H, int W);  // M-tiles per image of the generic tiling
// Halo variant (3x3, stride 1): one 128B-swizzled [18][10][64 ch] patch per 64-channel block serves all nine taps.
constexpr int kHaloTh = 16, kHaloTw = 8;
// Work-list pair tile: the unit of work is four 8x8 tiles, each read as one [10][10][64 ch] patch (make_act_map with a
// (kListTile + 2)-square box)
constexpr int kListTile = 8;
bool make_act_map_halo(CUtensorMap* map, const void* base, int B, int H, int W, int C, int pitch, int fp16 = 0);
// Policy: use the halo variant when its fixed 16x8 tiling costs at most 10 % more tiles than the best generic
// tiling over all segments.
bool conv_prefer_halo(int taps, int stride, int block_n, int nseg, const int* Hs, const int* Ws);
// Taps-in-N variant (3x3, stride 1, cout_pad == 16): the nine taps become GEMM columns -- ONE [180 patch pixels] x [9 x 16]
// GEMM per 64-channel block instead of nine N = 16 GEMMs (an N = 16 wgmma runs far below the tensor-core rate), then the
// nine shifted partial sums are added from shared memory.  Weights: bf16 [9 * 16][cin_pad64] (row = tap * 16 + cout).
constexpr int kTapsN = 144;
bool make_weight_map_taps(CUtensorMap* map, const void* base, int cin_pad, int fp16 = 0);
bool conv_taps_eligible(int taps, int stride, int cout_pad, int nseg, const int* Hs, const int* Ws);
void conv_set_taps(int mode);
// N-split of under-filled launches (engine.cu Builder::conv): 1 on (default; DD3D_CONV_NSPLIT=0 turns it off), -1 = environment
bool conv_wstat_enabled();       // weight-stationary halo layers: on by default, DD3D_CONV_WSTAT=0 / conv_set_wstat(0) turn it off
void conv_set_wstat(int mode);   // 0 off, 1 on, -1 environment / default
bool conv_n_split_enabled();
void conv_set_n_split(int mode);  // 0 off, 1 on, -1 environment / default (on)
// Pair tile for halo layers whose cout_pad is a multiple of 128 (out_mode 0, not taps-in-N): when selected, sets p->pair,
// block_n = 128 and n_blocks = cout_pad / 128 (the caller then needs a weight map with 128-row boxes) and returns true.
// Needs the halo tiling of every segment set.  Default rule: also (tile pairs x n-blocks) >= num_sms, so small launches keep
// the 128-pixel tile and the N-split.  conv_set_pair / DD3D_CONV_PAIR=0: 0 off, 1 on wherever eligible, -1 default.
bool conv_select_pair(ConvParams* p, int cout_pad, int num_sms);
void conv_set_pair(int mode);
// Consumer-warpgroup skew (ConvParams::stagger): -1 the default rule of conv_finalize_params, >= 0 that many k-blocks
// (clamped to the same bound).  dd3d_set_conv_policy("stagger", v); for A/B runs and tests.
void conv_set_stagger(int mode);
// N tile of a layer with cout_pad output channels: cout_pad itself up to 256, 256 for multiples of 256, otherwise the
// largest multiple of 64 that is <= 256 and divides cout_pad (384 -> 192: every 64-channel store box stays inside its
// n-block).  0: no such tile (the width is refused).
int conv_block_n(int cout_pad);
// Fills num_stages / total_work / tile bookkeeping from the already-set fields.
void conv_finalize_params(ConvParams* p);
cudaError_t launch_conv(const ConvParams& p, int num_sms, cudaStream_t stream);

}  // namespace dd3d
