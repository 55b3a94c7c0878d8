// Quantized-communication codecs (sm_90a): what travels on the wire of the pooled / sequence embedding collectives when a
// `QCommsConfig` asks for less than fp32 (reference torchrec/distributed/fbgemm_qcomm_codec.py:31-254, fbgemm quantize_comm):
//
//   FP8 row-wise   per row of `row_dim` elements: e4m3 payload + one fp32 scale (amax / 448), layout [rows][row_dim + 4 bytes]
//   INT8 row-wise  per row: uint8 payload + fp32 scale + fp32 bias,                 layout [rows][row_dim + 8 bytes]
//   MX4            per group of 32 elements: one shared e8m0 exponent byte + 32 x e2m1 (4 bit) values, layout [groups][1 + 16 bytes]
//
// One warp per row (FP8 / INT8) or per 32-element group (MX4, one lane per element); amax / min / max through shuffles; encode and
// decode are single passes over the data. fp16 / bf16 codecs are plain casts (torch).
#include "common.cuh"
#include <cuda_fp8.h>

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---- FP8 (e4m3) row-wise ----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) qcomm_fp8_encode_kernel(const float* __restrict__ in, uint8_t* __restrict__ out, int64_t rows, int row_dim) {
  const int lane = threadIdx.x & 31;
  const int64_t r = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (r >= rows) return;
  const float* src = in + r * row_dim;
  float amax = 0.f;
  for (int i = lane; i < row_dim; i += 32) amax = fmaxf(amax, fabsf(src[i]));
  amax = warp_max(amax);
  const float scale = amax > 0.f ? amax / 448.f : 1.f;
  const float inv = 1.f / scale;
  uint8_t* dst = out + r * (int64_t) (row_dim + 4);
  for (int i = lane; i < row_dim; i += 32) {
    const __nv_fp8_e4m3 q(src[i] * inv);
    dst[i] = *reinterpret_cast<const uint8_t*>(&q);
  }
  if (lane == 0) memcpy(dst + row_dim, &scale, 4);
}

__global__ void __launch_bounds__(256) qcomm_fp8_decode_kernel(const uint8_t* __restrict__ in, float* __restrict__ out, int64_t rows, int row_dim) {
  const int lane = threadIdx.x & 31;
  const int64_t r = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (r >= rows) return;
  const uint8_t* src = in + r * (int64_t) (row_dim + 4);
  float scale;
  memcpy(&scale, src + row_dim, 4);
  float* dst = out + r * row_dim;
  for (int i = lane; i < row_dim; i += 32) {
    __nv_fp8_e4m3 q;
    *reinterpret_cast<uint8_t*>(&q) = src[i];
    dst[i] = static_cast<float>(q) * scale;
  }
}

// ---- INT8 row-wise (scale + bias) ----------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) qcomm_int8_encode_kernel(const float* __restrict__ in, uint8_t* __restrict__ out, int64_t rows, int row_dim) {
  const int lane = threadIdx.x & 31;
  const int64_t r = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (r >= rows) return;
  const float* src = in + r * row_dim;
  float lo = 3.4e38f, hi = -3.4e38f;
  for (int i = lane; i < row_dim; i += 32) { lo = fminf(lo, src[i]); hi = fmaxf(hi, src[i]); }
  lo = warp_min(lo);
  hi = warp_max(hi);
  const float scale = hi > lo ? (hi - lo) / 255.f : 1.f;
  const float inv = 1.f / scale;
  uint8_t* dst = out + r * (int64_t) (row_dim + 8);
  for (int i = lane; i < row_dim; i += 32) dst[i] = (uint8_t) fminf(fmaxf(rintf((src[i] - lo) * inv), 0.f), 255.f);
  if (lane == 0) { memcpy(dst + row_dim, &scale, 4); memcpy(dst + row_dim + 4, &lo, 4); }
}

__global__ void __launch_bounds__(256) qcomm_int8_decode_kernel(const uint8_t* __restrict__ in, float* __restrict__ out, int64_t rows, int row_dim) {
  const int lane = threadIdx.x & 31;
  const int64_t r = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (r >= rows) return;
  const uint8_t* src = in + r * (int64_t) (row_dim + 8);
  float scale, bias;
  memcpy(&scale, src + row_dim, 4);
  memcpy(&bias, src + row_dim + 4, 4);
  float* dst = out + r * row_dim;
  for (int i = lane; i < row_dim; i += 32) dst[i] = src[i] * scale + bias;
}

// ---- MX4: groups of 32 x e2m1 with one shared power-of-two scale (e8m0) ---------------------------------------------------------------
// e2m1 magnitudes: 0, 0.5, 1, 1.5, 2, 3, 4, 6. Shared exponent = floor(log2(amax)) - 2 so that amax lands in [4, 8) -> clamps to 6.
__device__ __forceinline__ uint32_t e2m1_encode(float x) {
  const float a = fabsf(x);
  uint32_t m;
  if (a < 0.25f) m = 0; else if (a < 0.75f) m = 1; else if (a < 1.25f) m = 2; else if (a < 1.75f) m = 3;
  else if (a < 2.5f) m = 4; else if (a < 3.5f) m = 5; else if (a < 5.f) m = 6; else m = 7;
  return m | (x < 0.f ? 8u : 0u);
}
__device__ __forceinline__ float e2m1_decode(uint32_t q) {
  const float tab[8] = {0.f, 0.5f, 1.f, 1.5f, 2.f, 3.f, 4.f, 6.f};
  const float v = tab[q & 7];
  return (q & 8) ? -v : v;
}

__global__ void __launch_bounds__(256) qcomm_mx4_encode_kernel(const float* __restrict__ in, uint8_t* __restrict__ out, int64_t n_groups, int64_t n) {
  const int lane = threadIdx.x & 31;
  const int64_t g = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (g >= n_groups) return;
  const int64_t i = g * 32 + lane;
  const float x = i < n ? in[i] : 0.f;
  const float amax = warp_max(fabsf(x));
  int e = amax > 0.f ? (int) floorf(log2f(amax)) - 2 : -127;
  e = e < -127 ? -127 : (e > 127 ? 127 : e);
  const uint32_t q = e2m1_encode(x * exp2f((float) -e));
  const uint32_t hi = __shfl_down_sync(0xffffffffu, q, 1);
  uint8_t* dst = out + g * 17;
  if ((lane & 1) == 0) dst[1 + (lane >> 1)] = (uint8_t) (q | (hi << 4));
  if (lane == 0) dst[0] = (uint8_t) (e + 127);
}

__global__ void __launch_bounds__(256) qcomm_mx4_decode_kernel(const uint8_t* __restrict__ in, float* __restrict__ out, int64_t n_groups, int64_t n) {
  const int lane = threadIdx.x & 31;
  const int64_t g = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (g >= n_groups) return;
  const uint8_t* src = in + g * 17;
  const float scale = exp2f((float) ((int) src[0] - 127));
  const uint8_t b = src[1 + (lane >> 1)];
  const uint32_t q = (lane & 1) ? (b >> 4) : (b & 15);
  const int64_t i = g * 32 + lane;
  if (i < n) out[i] = e2m1_decode(q) * scale;
}

// codec: 0 = fp8 row-wise, 1 = int8 row-wise, 2 = mx4.  encode: fp32 [rows, row_dim] -> bytes;  decode: bytes -> fp32.
TRB_API int64_t trb_qcomm_encoded_bytes(int codec, int64_t rows, int row_dim) {
  if (codec == 0) return rows * (int64_t) (row_dim + 4);
  if (codec == 1) return rows * (int64_t) (row_dim + 8);
  if (codec == 2) return ((rows * row_dim + 31) / 32) * 17;
  return -1;
}

TRB_API int trb_qcomm_encode(int codec, const float* in, void* out, int64_t rows, int row_dim, cudaStream_t stream) {
  if (rows == 0 || row_dim == 0) return 0;
  const int threads = 256;
  if (codec == 0 || codec == 1) {
    const unsigned blocks = (unsigned) ((rows * 32 + threads - 1) / threads);
    if (codec == 0) qcomm_fp8_encode_kernel<<<blocks, threads, 0, stream>>>(in, (uint8_t*) out, rows, row_dim);
    else qcomm_int8_encode_kernel<<<blocks, threads, 0, stream>>>(in, (uint8_t*) out, rows, row_dim);
  } else if (codec == 2) {
    const int64_t n = rows * row_dim, groups = (n + 31) / 32;
    qcomm_mx4_encode_kernel<<<(unsigned) ((groups * 32 + threads - 1) / threads), threads, 0, stream>>>(in, (uint8_t*) out, groups, n);
  } else {
    return -3;
  }
  TRB_CHECK_LAUNCH();
  return 0;
}

TRB_API int trb_qcomm_decode(int codec, const void* in, float* out, int64_t rows, int row_dim, cudaStream_t stream) {
  if (rows == 0 || row_dim == 0) return 0;
  const int threads = 256;
  if (codec == 0 || codec == 1) {
    const unsigned blocks = (unsigned) ((rows * 32 + threads - 1) / threads);
    if (codec == 0) qcomm_fp8_decode_kernel<<<blocks, threads, 0, stream>>>((const uint8_t*) in, out, rows, row_dim);
    else qcomm_int8_decode_kernel<<<blocks, threads, 0, stream>>>((const uint8_t*) in, out, rows, row_dim);
  } else if (codec == 2) {
    const int64_t n = rows * row_dim, groups = (n + 31) / 32;
    qcomm_mx4_decode_kernel<<<(unsigned) ((groups * 32 + threads - 1) / threads), threads, 0, stream>>>((const uint8_t*) in, out, groups, n);
  } else {
    return -3;
  }
  TRB_CHECK_LAUNCH();
  return 0;
}
