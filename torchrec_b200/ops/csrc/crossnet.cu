// Element-wise halves of the DCN-v2 cross layer  x_{l+1} = x_0 * u + x_l  (u = W_l (V_l x_l) + b_l comes out of the GEMM epilogue).
// In eager PyTorch the forward is 2 kernels over [B, D] bf16 tensors and the backward 4-6 more (mul, mul, add-into-grad ...): for the
// 3-layer, 3456-wide cross net of the DLRM-DCN benchmark that is a large share of the step, all HBM streaming. Here:
//   forward   y = x0 * u + xl                                   (3 reads, 1 write)
//   backward  gu = g * x0;  gx0 = g * u                         (3 reads, 2 writes; the gradient of xl is g itself, no kernel)
// bf16 storage, fp32 math, 16-byte vectors, grid-stride.
#include "common.cuh"

namespace {

__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    f[2 * i] = __uint_as_float(w[i] << 16);
    f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
  }
}

__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
    w[i] = *reinterpret_cast<uint32_t*>(&h);
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}

__global__ void __launch_bounds__(256) cross_fwd_kernel(const uint4* __restrict__ x0, const uint4* __restrict__ u, const uint4* __restrict__ xl,
                                                        uint4* __restrict__ y, int64_t nvec) {
  for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (int64_t) gridDim.x * blockDim.x) {
    const uint4 a = x0[i], b = u[i], c = xl[i];
    float fa[8], fb[8], fc[8], o[8];
    unpack8(a, fa);
    unpack8(b, fb);
    unpack8(c, fc);
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] = fmaf(fa[k], fb[k], fc[k]);
    y[i] = pack8(o);
  }
}

__global__ void __launch_bounds__(256) cross_bwd_kernel(const uint4* __restrict__ g, const uint4* __restrict__ x0, const uint4* __restrict__ u,
                                                        uint4* __restrict__ gu, uint4* __restrict__ gx0, int64_t nvec) {
  for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (int64_t) gridDim.x * blockDim.x) {
    const uint4 gv = g[i], a = x0[i], b = u[i];
    float fg[8], fa[8], fb[8], o[8], o2[8];
    unpack8(gv, fg);
    unpack8(a, fa);
    unpack8(b, fb);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      o[k] = fg[k] * fa[k];
      o2[k] = fg[k] * fb[k];
    }
    gu[i] = pack8(o);
    gx0[i] = pack8(o2);
  }
}

unsigned grid_for(int64_t nvec) {
  const int64_t b = (nvec + 255) / 256;
  const int64_t cap = (int64_t) trb_num_sms() * 8;
  return (unsigned) (b < cap ? b : cap);
}

}  // namespace

TRB_API int trb_cross_fwd(const void* x0, const void* u, const void* xl, void* y, int64_t n, cudaStream_t stream) {
  if (n == 0) return 0;
  if (n % 8) return -1;
  cross_fwd_kernel<<<grid_for(n / 8), 256, 0, stream>>>((const uint4*) x0, (const uint4*) u, (const uint4*) xl, (uint4*) y, n / 8);
  TRB_CHECK_LAUNCH();
  return 0;
}

TRB_API int trb_cross_bwd(const void* g, const void* x0, const void* u, void* gu, void* gx0, int64_t n, cudaStream_t stream) {
  if (n == 0) return 0;
  if (n % 8) return -1;
  cross_bwd_kernel<<<grid_for(n / 8), 256, 0, stream>>>((const uint4*) g, (const uint4*) x0, (const uint4*) u, (uint4*) gu, (uint4*) gx0, n / 8);
  TRB_CHECK_LAUNCH();
  return 0;
}
