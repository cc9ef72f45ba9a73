#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace dd3d {

// images: [B][3][Hs][Ws] uint8 or fp32 (each image top-left aligned, valid size sizes[b] = (h, w));
// All 16-bit activation buffers are bf16 or fp16 (trailing `fp16` flag, act16.cuh); typed __nv_bfloat16* either way.
// dst: [B][Hp][Wp][4] bf16, zero outside the valid region (pad AFTER normalisation, image_list.py:124-148).
cudaError_t launch_preprocess(const void* src, int src_is_u8, const int* d_sizes, int size_stride, __nv_bfloat16* dst,
                              int B, int Hs, int Ws, int Hp, int Wp, const float mean[3], const float std[3],
                              cudaStream_t stream, int fp16 = 0);

// DLA-34 front end fused (dla_front.cu): base_layer 7x7 -> level0 3x3 -> level1 3x3/s2 (+ 2x2 max-pool of the result), conv +
// BN + ReLU each, intermediates in shared memory.  in4: [B][H][W][4]; w0 [16][7][8][4], w1 [16][9][16], w2 [32][9][16] 16-bit;
// sb* = fp32 scale[cout] | bias[cout]; out [B][H/2][W/2][out_pitch]; pool (may be null) [B][H/4][W/4][pool_pitch].
cudaError_t launch_dla_front(const __nv_bfloat16* in4, const __nv_bfloat16* w0, const __nv_bfloat16* w1,
                             const __nv_bfloat16* w2, const float* sb0, const float* sb1, const float* sb2,
                             __nv_bfloat16* out, int out_pitch, __nv_bfloat16* pool, int pool_pitch, int B, int H, int W,
                             int num_sms, cudaStream_t stream, int fp16 = 0);

// VoVNet stem_1 (3x3 stride 2, 3 -> 64) on register fragments (stem_mma.cu).  w: 16-bit [64][3][4][4] (cout, ky, kx, c; kx = 3
// and c = 3 zero); sb: fp32 scale[64] | bias[64]; out: [B][ceil(H/2)][ceil(W/2)][out_pitch].  relu = 0: no ReLU after the
// folded affine (the raw conv output of a GroupNorm backbone).
cudaError_t launch_stem_s2_mma(const __nv_bfloat16* in4, const __nv_bfloat16* w, const float* sb, __nv_bfloat16* out,
                               int out_pitch, int B, int H, int W, int num_sms, cudaStream_t stream, int fp16 = 0,
                               int relu = 1);

cudaError_t launch_maxpool(const __nv_bfloat16* in, __nv_bfloat16* out, int B, int H, int W, int C, int in_pitch,
                           int Ho, int Wo, int out_pitch, int ksize, int num_sms, cudaStream_t stream, int fp16 = 0);

int ese_nsplit(int HW);
constexpr int kEseLaunches = 3;  // either form: pool (or reduce), fc, scale
// partial: [B][ese_nsplit(HW)][C] fp32 scratch, gate: [B][C] fp32 scratch.
cudaError_t launch_ese(const __nv_bfloat16* x, int x_pitch, const float* fc_w, const float* fc_b,
                       const __nv_bfloat16* identity, int id_pitch, __nv_bfloat16* out, int out_pitch, float* partial,
                       float* gate, int B, int HW, int C, int num_sms, cudaStream_t stream, int fp16 = 0);

// tile_partial: [B][T][C] fp32 rows written by the concat-conv epilogue (T = 4 * tiles per image); sums: [B][C] scratch.
cudaError_t launch_ese_fused(const __nv_bfloat16* x, int x_pitch, const float* tile_partial, int T, const float* fc_w,
                             const float* fc_b, const __nv_bfloat16* identity, int id_pitch, __nv_bfloat16* out,
                             int out_pitch, float* sums, float* gate, int B, int HW, int C, int num_sms,
                             cudaStream_t stream, int fp16 = 0);

// Depthwise 3x3 conv, padding 1, stride 1 or 2 (dwconv.cu): in / out NHWC 16-bit with channel pitches, w 16-bit [9][C]
// (tap = r * 3 + s); fp32 accumulation in tap order, no bias / norm / activation.  C, both pitches multiples of 8.
int dwconv3x3_out_size(int n, int stride);
cudaError_t launch_dwconv3x3(const __nv_bfloat16* in, int B, int H, int W, int C, int in_pitch, const __nv_bfloat16* w,
                             int stride, __nv_bfloat16* out, int out_pitch, cudaStream_t stream, int fp16 = 0);

cudaError_t launch_relu(const __nv_bfloat16* x, __nv_bfloat16* out, size_t n_elems, int num_sms, cudaStream_t stream);

}  // namespace dd3d
