// GroupNorm(32, 256) of the FCOS towers and the FPN (group_norm.cu): statistics + apply over up to kMaxSeg maps per launch.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stddef.h>

#include "conv_igemm.cuh"  // kMaxSeg

namespace dd3d {

constexpr int kGnChannels = 256;  // 32 groups of 8 channels
constexpr int kGnChunk = 1024;    // pixels per statistics chunk (a function of the shape only: deterministic)

struct GroupNormSeg {
    const __nv_bfloat16* in = nullptr;   // [B][H][W][in_pitch], channels [0, 256)
    __nv_bfloat16* out = nullptr;        // [B][H][W][out_pitch]; may equal `in`
    const __nv_bfloat16* res = nullptr;  // optional [B][res_H][res_W][res_pitch]: added as nearest-2x after the norm
    int H = 0, W = 0, in_pitch = 0, out_pitch = 0, res_pitch = 0, res_H = 0, res_W = 0;
    float2* part = nullptr;  // group_norm_scratch_bytes(B, H, W) bytes: (mean, M2) per (image, chunk, group)
    int nchunks = 0, cta0 = 0;  // set by launch_group_norm
};

struct GroupNormParams {
    GroupNormSeg seg[kMaxSeg];
    int nseg = 0, B = 0;
    const float* gamma = nullptr;  // fp32 [256]; nullptr: no normalisation (s = 1, b = 0)
    const float* beta = nullptr;
    int relu = 0, avg = 0, fp16 = 0;
};

int group_norm_chunks(int H, int W);
size_t group_norm_scratch_bytes(int B, int H, int W);
// One launch of the statistics kernel (skipped when gamma == nullptr) and one of the apply kernel over every segment.
cudaError_t launch_group_norm(GroupNormParams p, cudaStream_t stream);

}  // namespace dd3d
