// Sparse FCOS3D predictor (b3d_sparse.cu): the fused box3d 3x3 conv evaluated at the final 2-D candidates only.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "detect.cuh"

namespace dd3d {

struct B3dSparseLevel {
    const __nv_bfloat16* in;  // box3d tower output of the level, NHWC 16-bit [B][H][W][pitch], cin channels
    const __nv_bfloat16* w;   // fused predictor weights [n_pad][9][cin] (engine conv_layer layout; per level when PER_LEVEL_PREDICTORS)
    const float* scale;       // [n_pad] per-level epilogue (Scale folded)
    const float* bias;        // [n_pad] conv bias * scale (+ depth Offset)
    int H, W, pitch;
};

struct B3dSparseParams {
    B3dSparseLevel lvl[kLevels];
    const uint2* fin;           // [B][L][topk] (score bits, pixel * C + class): DecodeParams::fin
    const int32_t* cand_count;  // [B][L]
    float* rows;                // [B][L][topk][out_pitch] fp32, channel layout of a dense map pixel
    int num_levels;             // L: lvl[0 .. L) are read (DecodeParams::num_levels)
    int B, C, topk, n_pad, out_pitch, fp16;
    int cin;  // tower width (FE.FPN.OUT_CHANNELS): a multiple of 64 in [64, kB3dSparseMaxCin]
};

// widest fused predictor the kernel is instantiated for (14 n-tiles of 8: the 10 nuScenes classes); the engine keeps the dense
// predictor for models with more 3-D output channels
constexpr int kB3dSparseMaxN = 112;
constexpr int kB3dSparseMaxCin = 512;  // widest FPN the engine builds
cudaError_t launch_b3d_sparse(const B3dSparseParams& p, cudaStream_t stream);

// Class-gathered sparse FCOS3D predictor (b3d_gather.cu), for class-specific heads wider than kB3dSparseMaxN: the decode reads
// only the 11 channels {q * C + c} of a candidate's own class c (fcos3d.py:333-352), so each candidate gets exactly those,
// computed with the same per-channel arithmetic as b3d_sparse_kernel.  lvl[].w is the whole fused predictor [>= 11 C][9][cin],
// lvl[].scale / bias its [11 C] epilogue.  Output rows [B][L][topk][kB3dGatherPitch] fp32: channel q of the candidate's class
// at column q (the layout of a class-agnostic map pixel); columns 11..15 are not written.
constexpr int kB3dGatherPitch = 16;
constexpr int kB3dGatherMaxC = 128;  // DD3D_MAX_NUM_CLASSES
struct B3dGatherParams {
    B3dSparseLevel lvl[kLevels];
    const uint2* fin;           // [B][L][topk] (score bits, pixel * C + class): DecodeParams::fin
    const int32_t* cand_count;  // [B][L]
    float* rows;                // [B][L][topk][kB3dGatherPitch]
    int32_t* order;             // scratch [B][L][topk]: the slots of each (image, level), grouped by class
    int2* seg;                  // scratch [B][L][C]: (first entry in `order`, count) of each class
    int num_levels;             // L: lvl[0 .. L) are read (DecodeParams::num_levels)
    int B, C, topk, fp16, cin;
};
size_t b3d_gather_scratch_bytes(int B, int C, int topk, int num_levels = kLevels);
void b3d_gather_bind_scratch(B3dGatherParams* p, void* scratch);
constexpr int kB3dGatherLaunches = 2;  // class grouping + predictor
cudaError_t launch_b3d_gather(const B3dGatherParams& p, cudaStream_t stream);

// Sparse box3d tower (tower_tiles.cu): the sparse predictor reads the tower output only in the 3x3 neighbourhoods of the
// final candidates, so tower layer i of `depth` (0-based) is needed only at the candidates dilated by depth - i pixels
// (Chebyshev), clipped to the map.  tower_tiles_kernel lists, per layer, the conv tiles that meet that set; the tower convs
// then run the pair tile in work-list mode (ConvParams::tile_list) on exactly those 8x8 tiles (kListTile); every (image, level)
// list is padded to a multiple of 4 entries with the out-of-image tile, so that a work unit of four tiles never spans two
// levels or images.
//
// Sparse box2d tower: the decode reads the [box2d_reg | centerness] map only at the pixels of P, where some class passes the
// class-only threshold (class_passes, detect.cuh), and the predictor is a 3x3 conv of the last tower layer.  So list `depth`
// - 1 (the predictor's) holds the tiles that meet P, and tower layer i the tiles within depth - 1 - i of it.  Its seeds come
// from a pixel-parallel marking pass over the cls maps (launch_tower_mark), which lowers the tile distances in `dist`.  The
// predictor (the taps-in-N kernel) works on 16x8 tiles: its list (pred16) holds the 16x8 tiles one of whose two 8x8 halves
// meets P, unpadded.
//
// List i holds the tiles at distance <= reach - i from a seed: reach = depth for the box3d tower (its predictor reads 3x3
// neighbourhoods of the candidates), depth - 1 for the box2d tower and its predictor.
struct TowerTilesLevel {
    int H, W, th, tw, tiles_x, tiles_y;
    int stage_begin;  // first entry of this level's (image-major) per-image regions in a layer's staging / list area
    const float* cls;  // mark pass: cls map [B][H*W][cls_pitch] of the level
    int mark_begin;    // mark pass: first block (of grid.x) of this level
};
constexpr int kTowerTileFar = 0x3F3F3F3F;  // tile distance "no seed near": the 0x3F byte pattern (cudaMemset)
struct TowerTilesParams {
    TowerTilesLevel lvl[kLevels];
    const uint2* fin;           // seeds: DecodeParams::fin (nullptr: the distances of the mark pass in `dist`)
    const int32_t* cand_count;  // [B][L]
    int32_t* dist;              // mark pass: [cap] tile distances, (level, image) regions at the offsets of a layer's list;
                                // kTowerTileFar between launches (tower_tiles_kernel reads and resets them)
    int num_levels;             // L: lvl[0 .. L) (DecodeParams::num_levels)
    int B, C, topk, depth, reach;
    int pred16;                  // 1: list depth - 1 is the box2d predictor's, on 16x8 tiles (2 th x tw)
    int cls_pitch, mark_blocks;  // mark pass
    float thresh;                // mark pass: PRE_NMS_THRESH
    int cap;        // entries per layer: sum over levels of B * (tiles per image, rounded up to a multiple of 4)
    int max_tiles;  // largest tiles per image of a level (shared memory)
    uint32_t* stage;     // [depth][cap] per-(image, level) lists at fixed offsets
    int32_t* bl_count;   // [depth][L][B] entries of each (image, level) list
    int32_t* bl_pixels;  // [depth][L][B] in-map pixels of its real tiles
    uint32_t* list;      // [depth][cap] compacted lists, level-major, then image, then row-major tile: ConvParams::tile_list
    int32_t* count;      // [depth] entries of each compacted list: ConvParams::tile_count
    long long* pixels;   // [depth] in-map pixels of the listed tiles (the FLOPs the profile books)
    uint32_t* ticket;    // zero between launches; the last CTA to finish compacts and resets it
};
size_t tower_tiles_smem_bytes(int max_tiles);
constexpr int kTowerMarkThreads = 256;  // mark pass: head pixels per block (TowerTilesLevel::mark_begin)
cudaError_t launch_tower_mark(const TowerTilesParams& p, cudaStream_t stream);  // needs p.dist; then launch_tower_tiles
cudaError_t launch_tower_tiles(const TowerTilesParams& p, cudaStream_t stream);

}  // namespace dd3d
