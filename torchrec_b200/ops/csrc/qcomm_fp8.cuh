// The FP8 row-wise wire format, in one place: a group of R consecutive values travels as R e4m3 bytes plus one fp32 scale.
//
//   amax  = max |v| over the group
//   scale = amax > 0 ? amax / 448 : 1
//   q     = e4m3(v * (1 / scale))        round to nearest even, saturating to +-448
//   v'    = float(q) * scale
//
// The codec kernels of qcomm.cu (portable collectives) and the quantizing stores of the NVLink plane (tbe_fwd.cu, peer_mem.cu)
// all use these helpers, so a value sent either way decodes to the same bits.
#pragma once
#include <cuda_fp8.h>

#include "common.cuh"

__device__ __forceinline__ float trb_fp8_scale(float amax) { return amax > 0.f ? amax / 448.f : 1.f; }

__device__ __forceinline__ float trb_fp8_abs_max4(float4 v) { return fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))); }

// two values -> two e4m3 bytes (a in the low byte)
__device__ __forceinline__ uint32_t trb_fp8_encode2(float a, float b, float inv) {
  return (uint32_t) __nv_cvt_float2_to_fp8x2(make_float2(a * inv, b * inv), __NV_SATFINITE, __NV_E4M3);
}

__device__ __forceinline__ uint8_t trb_fp8_encode(float v, float inv) { return (uint8_t) (trb_fp8_encode2(v, 0.f, inv) & 0xffu); }

// four values -> four e4m3 bytes, v.x in the lowest byte (the byte order of the payload in memory)
__device__ __forceinline__ uint32_t trb_fp8_encode4(float4 v, float inv) {
  return trb_fp8_encode2(v.x, v.y, inv) | (trb_fp8_encode2(v.z, v.w, inv) << 16);
}

__device__ __forceinline__ float trb_fp8_decode(uint32_t q, float scale) {
  __nv_fp8_e4m3 e;
  e.__x = (__nv_fp8_storage_t) (q & 0xffu);
  return static_cast<float>(e) * scale;
}

__device__ __forceinline__ float4 trb_fp8_decode4(uint32_t q, float scale) {
  return make_float4(trb_fp8_decode(q, scale), trb_fp8_decode(q >> 8, scale), trb_fp8_decode(q >> 16, scale), trb_fp8_decode(q >> 24, scale));
}

// values as they are after a store in dtype T (the wire dtype the FP8 groups are formed from)
template <typename T>
__device__ __forceinline__ float4 trb_round_to(float4 v);
template <>
__device__ __forceinline__ float4 trb_round_to<float>(float4 v) { return v; }
template <>
__device__ __forceinline__ float4 trb_round_to<__nv_bfloat16>(float4 v) {
  const float2 a = __bfloat1622float2(__floats2bfloat162_rn(v.x, v.y)), b = __bfloat1622float2(__floats2bfloat162_rn(v.z, v.w));
  return make_float4(a.x, a.y, b.x, b.y);
}
