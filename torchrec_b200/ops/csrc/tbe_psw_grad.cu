// Gradient of the pooled table-batched lookup w.r.t. the per-sample weights (sm_90a):
//     d psw[i] = < grad_out[bag(i)][cols of f] , W[idx[i]] >     (x 1/L for MEAN pooling)
// One warp per bag keeps the bag's gradient row in registers and streams the bag's table rows through it;
// gradient rows may live on NVLink peers (same addressing as the fused backward). Must run BEFORE the fused
// backward + optimizer mutates the table rows. Parity: fbgemm's `indice_weights` gradient, consumed by the
// feature processors (reference torchrec/distributed/fp_embeddingbag.py:152-161, modules/feature_processor_.py:78).
#include "common.cuh"

struct PswGradParams {
  const void* weights;
  const int64_t* feat_woff;
  const int64_t* feat_rows;
  const int32_t* feat_dim;
  const int32_t* feat_col;
  TrbSrcView src;
  TrbPeerPtrs grad;
  int64_t grad_stride;
  float* out;  // [n]
  int32_t B, B_local, F, mean;
};

template <typename W, typename G, int MAXV>
__global__ void __launch_bounds__(256) tbe_psw_grad_kernel(const PswGradParams p) {
  const int lane = threadIdx.x & 31;
  const int64_t bag = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (bag >= (int64_t) p.F * p.B) return;
  const int f = (int) (bag / p.B);
  const int b = (int) (bag - (int64_t) f * p.B);
  int64_t pos_base;
  const int64_t oi = trb_src_off_index(p.src, f, b, &pos_base);
  const int64_t start = pos_base + trb_ld_idx(p.src.offsets, oi, p.src.off64);
  const int64_t end = pos_base + trb_ld_idx(p.src.offsets, oi + 1, p.src.off64);
  if (end <= start) return;
  const int D = p.feat_dim[f];
  const int nvec = D >> 2;
  const int64_t rows = p.feat_rows[f];
  const W* __restrict__ wbase = reinterpret_cast<const W*>(p.weights) + p.feat_woff[f];
  const int s = b / p.B_local;
  const int bl = b - s * p.B_local;
  const G* g = reinterpret_cast<const G*>(p.grad.p[s]) + (int64_t) bl * p.grad_stride + p.feat_col[f];
  float4 gr[MAXV];
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int vi = lane + k * 32;
    gr[k] = (vi < nvec) ? Vec4<G>::ld(g + vi * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const float scale = p.mean ? 1.f / (float) (end - start) : 1.f;
  for (int64_t i = start; i < end; ++i) {
    const int64_t idx = trb_ld_idx(p.src.indices, i, p.src.idx64);
    float acc = 0.f;
    if (idx >= 0 && idx < rows) {
      const W* row = wbase + idx * D;
#pragma unroll
      for (int k = 0; k < MAXV; ++k) {
        const int vi = lane + k * 32;
        if (vi < nvec) {
          const float4 w = Vec4<W>::ld_nc(row + vi * 4);
          acc += w.x * gr[k].x + w.y * gr[k].y + w.z * gr[k].z + w.w * gr[k].w;
        }
      }
    }
    acc = warp_sum(acc);
    if (lane == 0) p.out[i] = acc * scale;
  }
}

template <typename W, typename G>
static int launch_psw(const PswGradParams& p, int max_dim, cudaStream_t stream) {
  const int64_t n_bags = (int64_t) p.F * p.B;
  if (n_bags == 0) return 0;
  const int threads = 256;
  const unsigned blocks = (unsigned) ((n_bags * 32 + threads - 1) / threads);
  const int nvec = max_dim / 4;
  if (nvec <= 32) tbe_psw_grad_kernel<W, G, 1><<<blocks, threads, 0, stream>>>(p);
  else if (nvec <= 128) tbe_psw_grad_kernel<W, G, 4><<<blocks, threads, 0, stream>>>(p);
  else if (nvec <= 512) tbe_psw_grad_kernel<W, G, 16><<<blocks, threads, 0, stream>>>(p);
  else return -2;
  TRB_CHECK_LAUNCH();
  return 0;
}

TRB_API int trb_tbe_psw_grad_ms(const void* weights, int w_dtype, const int64_t* feat_woff, const int64_t* feat_rows, const int32_t* feat_dim,
                                const int32_t* feat_col, const void* indices, int idx64, const void* offsets, int off64, int n_src, int64_t idx_stride,
                                int64_t off_stride, void* const* grad_ptrs, int n_grad, int grad_dtype, int64_t grad_stride, float* out, int B,
                                int B_local, int F, int max_dim, int mean, cudaStream_t stream) {
  if (n_grad < 1 || n_grad > TRB_MAX_PEERS) return -1;
  if (n_src < 1 || B % n_src != 0) return -4;
  PswGradParams p;
  p.weights = weights; p.feat_woff = feat_woff; p.feat_rows = feat_rows; p.feat_dim = feat_dim; p.feat_col = feat_col;
  p.src.indices = indices; p.src.offsets = offsets; p.src.psw = nullptr; p.src.idx_stride = idx_stride; p.src.off_stride = off_stride;
  p.src.n_src = n_src; p.src.src_B = B / n_src; p.src.idx64 = idx64; p.src.off64 = off64;
  p.grad_stride = grad_stride; p.out = out;
  for (int i = 0; i < n_grad; ++i) p.grad.p[i] = grad_ptrs[i];
  p.B = B; p.B_local = B_local; p.F = F; p.mean = mean;
#define PSW_CASE(WD, WT, GD, GT) if (w_dtype == WD && grad_dtype == GD) return launch_psw<WT, GT>(p, max_dim, stream);
  PSW_CASE(TRB_F32, float, TRB_F32, float)
  PSW_CASE(TRB_F32, float, TRB_BF16, __nv_bfloat16)
  PSW_CASE(TRB_BF16, __nv_bfloat16, TRB_BF16, __nv_bfloat16)
  PSW_CASE(TRB_BF16, __nv_bfloat16, TRB_F32, float)
  PSW_CASE(TRB_F16, __half, TRB_F16, __half)
  PSW_CASE(TRB_F16, __half, TRB_F32, float)
#undef PSW_CASE
  return -3;
}

TRB_API int trb_tbe_psw_grad(const void* weights, int w_dtype, const int64_t* feat_woff, const int64_t* feat_rows, const int32_t* feat_dim,
                             const int32_t* feat_col, const void* indices, int idx64, const void* offsets, int off64, void* const* grad_ptrs,
                             int n_grad, int grad_dtype, int64_t grad_stride, float* out, int B, int B_local, int F, int max_dim, int mean,
                             cudaStream_t stream) {
  return trb_tbe_psw_grad_ms(weights, w_dtype, feat_woff, feat_rows, feat_dim, feat_col, indices, idx64, offsets, off64, 1, 0, 0, grad_ptrs, n_grad,
                             grad_dtype, grad_stride, out, B, B_local, F, max_dim, mean, stream);
}
