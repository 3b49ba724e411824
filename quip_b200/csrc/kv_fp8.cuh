// The e4m3 KV-cache format (include/quip_b200.h): one warp quantizes a head vector, and e4m3 bytes convert exactly to
// fp16.  Shared by the decode / extend kernels (attn_decode.cu) and the prefill kernels (attn_prefill.cu), so every
// writer of the cache rounds by the same rule.
#pragma once
#include <cuda_fp8.h>

#include "common.cuh"

namespace quip {

constexpr float E4M3_MAX = 448.f;

union AH8 {
  uint4 v;
  __half2 h2[4];
};

// One warp quantizes the head vector x (HD fp16 values): lane l takes elements l*HD/32 .. (l+1)*HD/32 - 1 and returns
// their e4m3 bytes (element l*HD/32 + i in byte i); every lane gets the scale.
template <int HD>
__device__ __forceinline__ uint32_t e4m3_quantize_warp(const __half* __restrict__ x, int lane, float& s) {
  constexpr int E = HD / 32;   // 2 or 4
  float f[E];
  const __half2* x2 = reinterpret_cast<const __half2*>(x) + lane * (E / 2);
#pragma unroll
  for (int i = 0; i < E / 2; ++i) {
    const float2 p = __half22float2(x2[i]);
    f[2 * i] = p.x;
    f[2 * i + 1] = p.y;
  }
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < E; ++i) amax = fmaxf(amax, fabsf(f[i]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  s = amax == 0.f ? 1.f : amax / E4M3_MAX;
  uint32_t w = 0;
#pragma unroll
  for (int i = 0; i < E / 2; ++i) {
    const __nv_fp8x2_storage_t p =
        __nv_cvt_float2_to_fp8x2(make_float2(f[2 * i] / s, f[2 * i + 1] / s), __NV_SATFINITE, __NV_E4M3);
    w |= (uint32_t)p << (16 * i);
  }
  return w;
}

// the bytes of e4m3_quantize_warp to the HD-byte slot dst
template <int HD>
__device__ __forceinline__ void e4m3_store_warp(uint8_t* dst, int lane, uint32_t w) {
  if constexpr (HD == 128) reinterpret_cast<uint32_t*>(dst)[lane] = w;
  else reinterpret_cast<uint16_t*>(dst)[lane] = (uint16_t)w;
}

// 8 e4m3 bytes -> 8 fp16 (exact)
__device__ __forceinline__ uint4 e4m3x8_to_h8(const uint2& u) {
  AH8 t;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint32_t w = i < 2 ? u.x : u.y;
    t.h2[i] = __half2(__nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)((w >> (16 * (i & 1))) & 0xFFFFu), __NV_E4M3));
  }
  return t.v;
}

}  // namespace quip
