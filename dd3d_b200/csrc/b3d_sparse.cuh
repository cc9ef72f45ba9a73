// Sparse FCOS3D predictor (b3d_sparse.cu): the fused box3d 3x3 conv evaluated at the final 2-D candidates only.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "detect.cuh"

namespace dd3d {

struct B3dSparseLevel {
    const __nv_bfloat16* in;  // box3d tower output of the level, NHWC 16-bit [B][H][W][pitch], 256 channels
    const __nv_bfloat16* w;   // fused predictor weights [n_pad][9][256] (engine conv_layer layout; per level when PER_LEVEL_PREDICTORS)
    const float* scale;       // [n_pad] per-level epilogue (Scale folded)
    const float* bias;        // [n_pad] conv bias * scale (+ depth Offset)
    int H, W, pitch;
};

struct B3dSparseParams {
    B3dSparseLevel lvl[kLevels];
    const uint2* fin;           // [B][L][topk] (score bits, pixel * C + class): DecodeParams::fin
    const int32_t* cand_count;  // [B][L]
    float* rows;                // [B][L][topk][out_pitch] fp32, channel layout of a dense map pixel
    int B, C, topk, n_pad, out_pitch, fp16;
};

// widest fused predictor the kernel is instantiated for (14 n-tiles of 8: the 10 nuScenes classes); the engine keeps the dense
// predictor for models with more 3-D output channels
constexpr int kB3dSparseMaxN = 112;
cudaError_t launch_b3d_sparse(const B3dSparseParams& p, cudaStream_t stream);

// Sparse box3d tower (tower_tiles.cu): the sparse predictor reads the tower output only in the 3x3 neighbourhoods of the
// final candidates, so tower layer i of `depth` (0-based) is needed only at the candidates dilated by depth - i pixels
// (Chebyshev), clipped to the map.  tower_tiles_kernel lists, per layer, the conv tiles that meet that set; the tower convs
// then run the pair tile in work-list mode (ConvParams::tile_list) on exactly those tiles; every (image, level) list is
// padded to an even length with an out-of-image tile, so that a pair never spans two levels.
struct TowerTilesLevel {
    int H, W, th, tw, tiles_x, tiles_y;
    int stage_begin;  // first entry of this level's (image-major) per-image regions in a layer's staging / list area
};
struct TowerTilesParams {
    TowerTilesLevel lvl[kLevels];
    const uint2* fin;           // DecodeParams::fin
    const int32_t* cand_count;  // [B][L]
    int B, C, topk, depth;
    int cap;        // entries per layer: sum over levels of B * (tiles per image, rounded up to even)
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
cudaError_t launch_tower_tiles(const TowerTilesParams& p, cudaStream_t stream);

}  // namespace dd3d
