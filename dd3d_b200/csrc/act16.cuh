// 16-bit activation / weight storage of the engine: bf16 (default) or fp16 (dd3d_model_desc.act_dtype, the reference's
// mixed-precision path is fp16 autocast, scripts/train.py:121).  Layouts and kernels are identical; only the conversion
// instructions, the wgmma operand type and the TMA element type differ, selected by a template flag or a warp-uniform flag.
// Buffers are typed __nv_bfloat16* throughout as "opaque 16-bit elements".
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <string.h>

namespace dd3d {

__device__ __forceinline__ uint32_t pack2_bf16(float a, float b) {
    __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ uint32_t pack2_f16(float a, float b) {
    __half2 v = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ uint32_t pack2_act(float a, float b, int fp16) {
    return fp16 ? pack2_f16(a, b) : pack2_bf16(a, b);
}
// ReLU fused into the conversion (cvt.rn.relu: negative results and -0 become +0): same value as rounding max(x, 0)
template <bool FP16>
__device__ __forceinline__ uint32_t pack2_relu(float a, float b) {
    uint32_t r;
    if (FP16) {
        asm("cvt.rn.relu.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
    } else {
        asm("cvt.rn.relu.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
    }
    return r;
}
__device__ __forceinline__ float2 unpack2_bf16(uint32_t u) {
    return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u));
}
__device__ __forceinline__ float2 unpack2_f16(uint32_t u) { return __half22float2(*reinterpret_cast<__half2*>(&u)); }
__device__ __forceinline__ float2 unpack2_act(uint32_t u, int fp16) { return fp16 ? unpack2_f16(u) : unpack2_bf16(u); }

// host: fp32 -> 16-bit storage, round to nearest even (matches the device conversions and torch .to(dtype))
inline uint16_t host_f32_to_bf16(float f) {
    uint32_t u;
    memcpy(&u, &f, 4);
    if ((u & 0x7fffffffu) > 0x7f800000u) return static_cast<uint16_t>((u >> 16) | 0x40);
    const uint32_t lsb = (u >> 16) & 1u;
    u += 0x7fffu + lsb;
    return static_cast<uint16_t>(u >> 16);
}
inline uint16_t host_f32_to_f16(float f) {
    const __half h = __float2half_rn(f);  // host-callable (software path in cuda_fp16.hpp)
    uint16_t r;
    memcpy(&r, &h, 2);
    return r;
}
inline uint16_t host_f32_to_act(float f, int fp16) { return fp16 ? host_f32_to_f16(f) : host_f32_to_bf16(f); }

}  // namespace dd3d
