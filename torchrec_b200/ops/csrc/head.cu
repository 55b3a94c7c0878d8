// Fused model head for binary CTR models (sm_90a): the final Linear(K -> 1) and BCE-with-logits (mean) loss.
//
// In the reference the DLRM head is ~25 small library kernels per step (bf16->fp32 cast, gemv, sigmoid / log-sigmoid /
// mul / add / mean for the loss, their backward twins, split-K gemv for the weight gradient, ReLU mask of the last hidden
// layer: reference models/dlrm.py:227-239 + nn.BCEWithLogitsLoss). Each is launch-latency bound at batch 32k. Here:
//   trb_rowdot_fwd   logits[b] = <x[b, :], w> + bias                              (one warp per row, bf16 x, fp32 w)
//   trb_bce_fwd_bwd  loss = mean(max(z,0) - z*y + log1p(exp(-|z|))),  dz = (sigmoid(z) - y) / B        (one pass)
//   trb_rowdot_bwd   dx[b, :] = dz[b] * w (* [x>0] : ReLU mask of the producing layer), dw += dz[b] * x[b, :], db += dz[b]
#include "common.cuh"

__global__ void __launch_bounds__(256) rowdot_fwd_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx, const float* __restrict__ w, const float* __restrict__ bias,
                                                         float* __restrict__ out, int B, int K) {
  const int lane = threadIdx.x & 31;
  const int64_t row = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (row >= B) return;
  const __nv_bfloat16* xr = x + row * ldx;
  float acc = 0.f;
  for (int k = lane * 8; k < K; k += 256) {
    const uint4 v = *reinterpret_cast<const uint4*>(xr + k);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
    const float4 w0 = *reinterpret_cast<const float4*>(w + k), w1 = *reinterpret_cast<const float4*>(w + k + 4);
    const float2 a = __bfloat1622float2(h[0]), b = __bfloat1622float2(h[1]), c = __bfloat1622float2(h[2]), d = __bfloat1622float2(h[3]);
    acc += a.x * w0.x + a.y * w0.y + b.x * w0.z + b.y * w0.w + c.x * w1.x + c.y * w1.y + d.x * w1.z + d.y * w1.w;
  }
  acc = warp_sum(acc);
  if (lane == 0) out[row] = acc + (bias ? bias[0] : 0.f);
}

TRB_API int trb_rowdot_fwd(const void* x, int64_t ldx, const float* w, const float* bias, float* out, int B, int K, cudaStream_t stream) {
  if (B == 0) return 0;
  if (K % 8 || ldx % 8) return -2;
  rowdot_fwd_kernel<<<(unsigned) (((int64_t) B * 32 + 255) / 256), 256, 0, stream>>>((const __nv_bfloat16*) x, ldx, w, bias, out, B, K);
  TRB_CHECK_LAUNCH();
  return 0;
}

// labels may be float or int64/int32 (lab_kind 0 float32, 1 int64, 2 int32)
__global__ void __launch_bounds__(256) bce_fwd_bwd_kernel(const float* __restrict__ z, const void* __restrict__ labels, int lab_kind, float* __restrict__ loss,
                                                          float* __restrict__ dz, int B, float inv_b) {
  __shared__ float part[8];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  float l = 0.f;
  if (i < B) {
    const float x = z[i];
    const float y = lab_kind == 0 ? reinterpret_cast<const float*>(labels)[i]
                                  : (lab_kind == 1 ? (float) reinterpret_cast<const int64_t*>(labels)[i] : (float) reinterpret_cast<const int32_t*>(labels)[i]);
    const float e = __expf(-fabsf(x));
    l = fmaxf(x, 0.f) - x * y + log1pf(e);
    const float sig = x >= 0.f ? 1.f / (1.f + e) : e / (1.f + e);
    dz[i] = (sig - y) * inv_b;
  }
  l = warp_sum(l);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = l;
  __syncthreads();
  if (threadIdx.x < 8) {
    float s = part[threadIdx.x];
    s += __shfl_down_sync(0xffu, s, 4);
    s += __shfl_down_sync(0xffu, s, 2);
    s += __shfl_down_sync(0xffu, s, 1);
    if (threadIdx.x == 0) atomicAdd(loss, s * inv_b);
  }
}

TRB_API int trb_bce_fwd_bwd(const float* z, const void* labels, int lab_kind, float* loss, float* dz, int B, cudaStream_t stream) {
  TRB_CUDA(cudaMemsetAsync(loss, 0, sizeof(float), stream));
  if (B == 0) return 0;
  bce_fwd_bwd_kernel<<<(B + 255) / 256, 256, 0, stream>>>(z, labels, lab_kind, loss, dz, B, 1.f / (float) B);
  TRB_CHECK_LAUNCH();
  return 0;
}

// Each block handles a tile of rows; per-thread partial dw over its rows, reduced through shared memory, one atomicAdd per
// (block, k). dx is written with 16 B stores.
__global__ void __launch_bounds__(256) rowdot_bwd_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx, const float* __restrict__ dz, const float* __restrict__ w,
                                                         __nv_bfloat16* __restrict__ dx, int64_t lddx, float* __restrict__ dw, float* __restrict__ db, int B, int K,
                                                         int relu_mask, int rows_per_block, float gscale) {
  extern __shared__ float sdw[];  // [8 warps][K]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t r0 = (int64_t) blockIdx.x * rows_per_block;
  const int64_t r1 = min((int64_t) B, r0 + rows_per_block);
  // this lane owns columns [8*lane + 256*t, +8) for t < ceil(K/256) (K <= 2048 -> at most 8 slices)
  float acc[8][8];
#pragma unroll
  for (int t = 0; t < 8; ++t)
#pragma unroll
    for (int q = 0; q < 8; ++q) acc[t][q] = 0.f;
  float dbacc = 0.f;
  for (int64_t row = r0 + warp; row < r1; row += 8) {
    const float g = dz[row] * gscale;
    dbacc += g;
    const __nv_bfloat16* xr = x + row * ldx;
    __nv_bfloat16* dr = dx ? dx + row * lddx : nullptr;
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const int k = lane * 8 + t * 256;
      if (k < K) {
        const uint4 v = *reinterpret_cast<const uint4*>(xr + k);
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
        float xv[8];
#pragma unroll
        for (int q = 0; q < 4; ++q) { const float2 f = __bfloat1622float2(h[q]); xv[2 * q] = f.x; xv[2 * q + 1] = f.y; }
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[t][q] += g * xv[q];
        if (dr) {
          const float4 w0 = *reinterpret_cast<const float4*>(w + k), w1 = *reinterpret_cast<const float4*>(w + k + 4);
          const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
          uint4 o;
          __nv_bfloat162* oh = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            float a = g * wv[2 * q], b = g * wv[2 * q + 1];
            if (relu_mask) { a = xv[2 * q] > 0.f ? a : 0.f; b = xv[2 * q + 1] > 0.f ? b : 0.f; }
            oh[q] = __floats2bfloat162_rn(a, b);
          }
          *reinterpret_cast<uint4*>(dr + k) = o;
        }
      }
    }
  }
#pragma unroll
  for (int t = 0; t < 8; ++t) {
    const int k = lane * 8 + t * 256;
    if (k < K)
#pragma unroll
      for (int q = 0; q < 8; ++q) sdw[warp * K + k + q] = acc[t][q];
  }
  dbacc = (lane == 0) ? dbacc : 0.f;
  __syncthreads();
  for (int k = threadIdx.x; k < K; k += 256) {
    float s = 0.f;
#pragma unroll
    for (int w8 = 0; w8 < 8; ++w8) s += sdw[w8 * K + k];
    atomicAdd(dw + k, s);
  }
  if (db) {
    // one value per warp (lane 0) -> block sum
    __shared__ float sdb[8];
    if (lane == 0) sdb[warp] = dbacc;
    __syncthreads();
    if (threadIdx.x == 0) {
      float s = 0.f;
      for (int w8 = 0; w8 < 8; ++w8) s += sdb[w8];
      atomicAdd(db, s);
    }
  }
}

TRB_API int trb_rowdot_bwd(const void* x, int64_t ldx, const float* dz, const float* w, void* dx, int64_t lddx, float* dw, float* db, int B, int K, int relu_mask,
                           float gscale, cudaStream_t stream) {
  if (K % 8 || ldx % 8 || K > 2048 || (dx && lddx % 8)) return -2;
  TRB_CUDA(cudaMemsetAsync(dw, 0, sizeof(float) * K, stream));
  if (db) TRB_CUDA(cudaMemsetAsync(db, 0, sizeof(float), stream));
  if (B == 0) return 0;
  const int rows_per_block = 64;
  const unsigned blocks = (unsigned) ((B + rows_per_block - 1) / rows_per_block);
  const size_t smem = (size_t) 8 * K * sizeof(float);
  if (smem > 48 * 1024) TRB_CUDA(cudaFuncSetAttribute(rowdot_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem));
  rowdot_bwd_kernel<<<blocks, 256, smem, stream>>>((const __nv_bfloat16*) x, ldx, dz, w, (__nv_bfloat16*) dx, lddx, dw, db, B, K, relu_mask, rows_per_block, gscale);
  TRB_CHECK_LAUNCH();
  return 0;
}
