// FP8 (e4m3) paged KV cache: the one write / read definition every kernel uses (DESIGN.md section 2).
//
//   write  c = e4m3_rn_satfinite(float(bf16(x)) / scale)    fp32 division (IEEE), round to nearest even, saturate at +-448
//   read   dequant(c) = bf16(float(c) * scale)               e4m3 -> f16 -> f32 is exact; one fp32 multiply, one rounding
//
// `scale` is the per-layer k_scale / v_scale of vLLM (default 1.0).  A reader that dequantizes a row and then runs the
// bf16 arithmetic on it gives the bits of the bf16 kernel run on the dequantized cache.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cmath>
#include <cstdint>

namespace vita {

// host check of the entry points: scales are finite and positive
inline bool kv_fp8_scales_ok(float k_scale, float v_scale) {
    return std::isfinite(k_scale) && std::isfinite(v_scale) && k_scale > 0.0f && v_scale > 0.0f;
}

// two values -> 2 e4m3 bytes (a in the low byte)
__device__ __forceinline__ uint32_t kv_fp8_quant2(float a, float b, float scale) {
    const float qa = __fdiv_rn(a, scale), qb = __fdiv_rn(b, scale);
    uint16_t r;
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(qb), "f"(qa));   // first source -> upper byte
    return r;
}

__device__ __forceinline__ float kv_fp8_dequant_half(uint32_t h, float scale) {
    return __bfloat162float(__float2bfloat16(__half2float(__ushort_as_half(static_cast<unsigned short>(h))) * scale));
}

// 4 e4m3 bytes (byte i = element i) -> 4 dequantized values (bf16-exact floats)
__device__ __forceinline__ void kv_fp8_dequant4(uint32_t w, float scale, float* f) {
    uint32_t lo, hi;
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(lo) : "h"(static_cast<uint16_t>(w & 0xffffu)));
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(hi) : "h"(static_cast<uint16_t>(w >> 16)));
    f[0] = kv_fp8_dequant_half(lo & 0xffffu, scale);
    f[1] = kv_fp8_dequant_half(lo >> 16, scale);
    f[2] = kv_fp8_dequant_half(hi & 0xffffu, scale);
    f[3] = kv_fp8_dequant_half(hi >> 16, scale);
}

}  // namespace vita
