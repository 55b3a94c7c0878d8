// NVLink peer-memory substrate: symmetric buffers shared between the per-GPU processes of one
// NVLink domain (CUDA IPC), a device-side all-rank barrier and the small helper kernels the fused
// collectives need (staging reduce, cast-copy into a symmetric buffer).
//
// This replaces NCCL on the embedding hot paths: kernels receive the peers' buffer addresses and
// load/store them directly over NVSwitch.
// NCCL stays the control plane (handle exchange, DDP all-reduce, multi-node fallback).
#include "common.cuh"
#include "qcomm_fp8.cuh"
#include <cstring>
#include <cstdio>

TRB_API int trb_set_device(int dev) { return (int) cudaSetDevice(dev); }

TRB_API int trb_peer_alloc(void** ptr, size_t bytes) {
  TRB_CUDA(cudaMalloc(ptr, bytes));
  TRB_CUDA(cudaMemset(*ptr, 0, bytes));
  TRB_CUDA(cudaDeviceSynchronize());
  return 0;
}

TRB_API int trb_peer_free(void* ptr) { return (int) cudaFree(ptr); }

// handle is CUDA_IPC_HANDLE_SIZE (64) bytes
TRB_API int trb_ipc_get_handle(void* ptr, void* out_handle) {
  cudaIpcMemHandle_t h;
  TRB_CUDA(cudaIpcGetMemHandle(&h, ptr));
  memcpy(out_handle, &h, sizeof(h));
  return 0;
}

TRB_API int trb_ipc_open_handle(const void* handle, void** out_ptr) {
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, sizeof(h));
  TRB_CUDA(cudaIpcOpenMemHandle(out_ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return 0;
}

TRB_API int trb_ipc_close(void* ptr) { return (int) cudaIpcCloseMemHandle(ptr); }

TRB_API int trb_can_access_peer(int dev, int peer) {
  int ok = 0;
  if (cudaDeviceCanAccessPeer(&ok, dev, peer) != cudaSuccess) return 0;
  return ok;
}

// ------------------------------------------------------------------------------------------------
// Device-side barrier over all ranks of the domain.
//   signal pad of rank r : uint32 flags[W]; slot s is written only by rank s.
//   epoch                : device-resident counter on every rank, bumped by the kernel itself so
//                          the barrier can be captured in CUDA graphs.
// Thread t of the single CTA publishes the new epoch to peer t (after a system-scope fence so that
// every earlier store of this GPU — including peer stores of the previous kernels in the stream —
// is visible first), then spins until peer t's epoch arrived in the local pad.
// ------------------------------------------------------------------------------------------------
__global__ void trb_barrier_kernel(TrbPeerPtrs pads, uint32_t* epoch_counter, int rank, int W) {
  __shared__ uint32_t s_epoch;
  if (threadIdx.x == 0) {
    s_epoch = *epoch_counter + 1;
    *epoch_counter = s_epoch;
  }
  __syncthreads();
  const uint32_t epoch = s_epoch;
  const int t = threadIdx.x;
  if (t < W) {
    __threadfence_system();
    uint32_t* remote = reinterpret_cast<uint32_t*>(pads.p[t]) + rank;
    st_release_sys(remote, epoch);
    const uint32_t* local = reinterpret_cast<const uint32_t*>(pads.p[rank]) + t;
    unsigned long long spins = 0;
    while ((int32_t) (ld_acquire_sys(local) - epoch) < 0) {
      __nanosleep(40);
      if (++spins > 250000000ull) {  // ~10 s: a peer never arrived -> fail loudly instead of hanging the GPU
        printf("[trb200] barrier timeout: rank %d waiting for rank %d (epoch %u, seen %u)\n", rank, t, epoch, ld_relaxed_sys(local));
        __trap();
      }
    }
  }
  __syncthreads();
  __threadfence_system();
}

TRB_API int trb_barrier(void* const* pad_ptrs, int W, int rank, uint32_t* epoch_counter, cudaStream_t stream) {
  if (W < 1 || W > TRB_MAX_PEERS) return -1;
  TrbPeerPtrs pads;
  for (int i = 0; i < TRB_MAX_PEERS; ++i) pads.p[i] = i < W ? pad_ptrs[i] : nullptr;
  trb_barrier_kernel<<<1, 32, 0, stream>>>(pads, epoch_counter, rank, W);
  TRB_CHECK_LAUNCH();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Staging reduce (row-wise "reduce-scatter" tail): out[b, c] (+)= sum_{j in contributors(c)} slab_j[b, c]
//   staging : [W][B][stride] (slab j written by rank j's lookup kernel over NVLink)
//   col_mask: [n_cols] uint32 bitmask of contributing ranks per column (0 -> column untouched)
// ------------------------------------------------------------------------------------------------
template <typename S, typename O>
__global__ void __launch_bounds__(256)
trb_staging_reduce_kernel(const S* __restrict__ staging, O* __restrict__ out, const uint32_t* __restrict__ col_mask, int B,
                          int n_cols, int64_t stride, int64_t out_stride, int64_t slab, int W) {
  const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;  // vector index
  const int vec_cols = n_cols >> 2;
  if (i >= (int64_t) B * vec_cols) return;
  const int b = (int) (i / vec_cols);
  const int c = (int) (i - (int64_t) b * vec_cols) << 2;
  const uint32_t m = col_mask[c];
  if (m == 0) return;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int j = 0; j < W; ++j) {
    if (m & (1u << j)) acc = f4_add(acc, Vec4<S>::ld(staging + j * slab + (int64_t) b * stride + c));
  }
  Vec4<O>::st(out + (int64_t) b * out_stride + c, acc);
}

TRB_API int trb_staging_reduce(const void* staging, int s_dtype, void* out, int o_dtype, const uint32_t* col_mask, int B, int n_cols,
                               int64_t stride, int64_t out_stride, int64_t slab, int W, cudaStream_t stream) {
  const int64_t n = (int64_t) B * (n_cols / 4);
  if (n == 0) return 0;
  const int threads = 256;
  const unsigned blocks = (unsigned) ((n + threads - 1) / threads);
#define TRB_SR(SC, ST, OC, OT)                                                                                        \
  if (s_dtype == SC && o_dtype == OC) {                                                                               \
    trb_staging_reduce_kernel<ST, OT><<<blocks, threads, 0, stream>>>((const ST*) staging, (OT*) out, col_mask, B,     \
                                                                        n_cols, stride, out_stride, slab, W);          \
    TRB_CHECK_LAUNCH();                                                                                                \
    return 0;                                                                                                          \
  }
  TRB_SR(TRB_F32, float, TRB_F32, float)
  TRB_SR(TRB_BF16, __nv_bfloat16, TRB_F32, float)
  TRB_SR(TRB_BF16, __nv_bfloat16, TRB_BF16, __nv_bfloat16)
  TRB_SR(TRB_F32, float, TRB_BF16, __nv_bfloat16)
#undef TRB_SR
  return -3;
}

// Compact-staging variant used by the sparse plane: the staging slabs hold ONLY the columns of row-sharded tables
// (`n_cols` of them, slab j = partial sums computed by rank j); staged column c lands in output column dst_col[c].
// Memory is W x B x (row-sharded columns) instead of W full [B, sum D] slabs.
template <typename S, typename O>
__global__ void __launch_bounds__(256)
trb_staging_reduce_cols_kernel(const S* __restrict__ staging, O* __restrict__ out, const uint32_t* __restrict__ col_mask,
                               const int32_t* __restrict__ dst_col, int B, int n_cols, int64_t stride, int64_t out_stride, int64_t slab, int W) {
  const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
  const int vec_cols = n_cols >> 2;
  if (i >= (int64_t) B * vec_cols) return;
  const int b = (int) (i / vec_cols);
  const int c = (int) (i - (int64_t) b * vec_cols) << 2;
  const uint32_t m = col_mask[c];
  if (m == 0) return;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int j = 0; j < W; ++j) {
    if (m & (1u << j)) acc = f4_add(acc, Vec4<S>::ld(staging + j * slab + (int64_t) b * stride + c));
  }
  Vec4<O>::st(out + (int64_t) b * out_stride + dst_col[c], acc);
}

TRB_API int trb_staging_reduce_cols(const void* staging, int s_dtype, void* out, int o_dtype, const uint32_t* col_mask, const int32_t* dst_col, int B,
                                    int n_cols, int64_t stride, int64_t out_stride, int64_t slab, int W, cudaStream_t stream) {
  const int64_t n = (int64_t) B * (n_cols / 4);
  if (n == 0) return 0;
  const int threads = 256;
  const unsigned blocks = (unsigned) ((n + threads - 1) / threads);
#define TRB_SRC(SC, ST, OC, OT)                                                                                            \
  if (s_dtype == SC && o_dtype == OC) {                                                                                    \
    trb_staging_reduce_cols_kernel<ST, OT><<<blocks, threads, 0, stream>>>((const ST*) staging, (OT*) out, col_mask,      \
                                                                             dst_col, B, n_cols, stride, out_stride, slab, W); \
    TRB_CHECK_LAUNCH();                                                                                                     \
    return 0;                                                                                                               \
  }
  TRB_SRC(TRB_F32, float, TRB_F32, float)
  TRB_SRC(TRB_BF16, __nv_bfloat16, TRB_BF16, __nv_bfloat16)
#undef TRB_SRC
  return -3;
}

// Single-process multi-GPU harnesses (tools/bench_peer_copy.py, tests): let kernels on `dev` address memory of `peer`.
TRB_API int trb_enable_peer_access(int dev, int peer) {
  int cur = 0;
  TRB_CUDA(cudaGetDevice(&cur));
  TRB_CUDA(cudaSetDevice(dev));
  cudaError_t e = cudaDeviceEnablePeerAccess(peer, 0);
  if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); e = cudaSuccess; }
  cudaSetDevice(cur);
  return (int) e;
}

// ------------------------------------------------------------------------------------------------
// Strided cast-copy: dst[b, c] = (D) src[b, c] * scale   (used to stage gradients into the symmetric
// buffer the peers pull from, with the 1/W gradient division and the wire dtype cast fused in)
// ------------------------------------------------------------------------------------------------
template <typename S, typename D>
__global__ void __launch_bounds__(256)
trb_cast_copy_kernel(const S* __restrict__ src, D* __restrict__ dst, int64_t rows, int cols, int64_t src_stride, int64_t dst_stride, float scale) {
  const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
  const int vec_cols = cols >> 2;
  if (i >= rows * vec_cols) return;
  const int64_t r = i / vec_cols;
  const int c = (int) (i - r * vec_cols) << 2;
  float4 v = Vec4<S>::ld(src + r * src_stride + c);
  if (scale != 1.f) v = f4_scale(v, scale);
  Vec4<D>::st(dst + r * dst_stride + c, v);
}

TRB_API int trb_cast_copy(const void* src, int s_dtype, void* dst, int d_dtype, int64_t rows, int cols, int64_t src_stride,
                          int64_t dst_stride, float scale, cudaStream_t stream) {
  const int64_t n = rows * (cols / 4);
  if (n == 0) return 0;
  const int threads = 256;
  const unsigned blocks = (unsigned) ((n + threads - 1) / threads);
#define TRB_CC(SC, ST, DC, DT)                                                                                                   \
  if (s_dtype == SC && d_dtype == DC) {                                                                                          \
    trb_cast_copy_kernel<ST, DT><<<blocks, threads, 0, stream>>>((const ST*) src, (DT*) dst, rows, cols, src_stride, dst_stride, scale); \
    TRB_CHECK_LAUNCH();                                                                                                           \
    return 0;                                                                                                                     \
  }
  TRB_CC(TRB_F32, float, TRB_F32, float)
  TRB_CC(TRB_F32, float, TRB_BF16, __nv_bfloat16)
  TRB_CC(TRB_BF16, __nv_bfloat16, TRB_F32, float)
  TRB_CC(TRB_BF16, __nv_bfloat16, TRB_BF16, __nv_bfloat16)
#undef TRB_CC
  return -3;
}

// ---------------------------------------------------------------------------------------------------------------
// Gradient push (backward "all-to-all" as posted NVLink stores): every rank scatters the column blocks of its local
// gradient [B_local, total_cols] to the ranks that own the corresponding table shards, into THEIR gradient inbox
// [W * B_local, pitch] at rows [src_rank * B_local, ...). Chunks of 4 elements are described by a small device table
// (dst rank, src col, dst col). Posted remote writes pipeline far deeper than the remote row *reads* of a pull design
// (a peer load is a full NVLink round trip), and the fused backward afterwards only touches local HBM.
// Parity: the backward all_to_all_single of the pooled output dist (reference comm_ops.py:1581-1646).
// ---------------------------------------------------------------------------------------------------------------
// VEC = elements per chunk (4 or 8). 8-element chunks move 16 B per thread for bf16 gradients.
//
// PERSISTENT, narrow launch: the kernel is NVLink-bound (posted peer stores), it needs bytes in flight, not thread slots. The
// first version launched one thread per chunk (53 k blocks for a DLRM batch): those blocks filled every thread slot of every SM for
// the whole transfer and starved the weight-gradient GEMMs that are meant to run beside it.
// Now ~2 CTAs per SM walk the chunks with a grid stride, UNR independent 16 B loads in flight per thread before the stores.
template <typename S, typename D, int VEC, int UNR>
__global__ void __launch_bounds__(256)
trb_grad_push_kernel(const S* __restrict__ src, int64_t src_stride, const int32_t* __restrict__ chunks, int n_chunks, TrbPeerPtrs dst, int64_t dst_pitch,
                     int64_t row_base, int B_local, float scale) {
  const int64_t total = (int64_t) B_local * n_chunks;
  const int64_t stride = (int64_t) gridDim.x * blockDim.x;
  for (int64_t i0 = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i0 < total; i0 += stride * UNR) {
    const S* sp[UNR];
    D* dp[UNR];
    bool ok[UNR];
#pragma unroll
    for (int u = 0; u < UNR; ++u) {
      const int64_t i = i0 + u * stride;
      ok[u] = i < total;
      const int64_t ii = ok[u] ? i : i0;
      const int64_t b = total < 0x7fffffffLL ? (int64_t) ((uint32_t) ii / (uint32_t) n_chunks) : ii / n_chunks;
      const int c = (int) (ii - b * n_chunks);
      const int rank = chunks[3 * c], sc = chunks[3 * c + 1], dc = chunks[3 * c + 2];
      sp[u] = src + b * src_stride + sc;
      dp[u] = reinterpret_cast<D*>(dst.p[rank]) + (row_base + b) * dst_pitch + dc;
    }
    if constexpr (VEC == 8 && sizeof(S) == 2 && sizeof(D) == 2) {
      uint4 v[UNR];
#pragma unroll
      for (int u = 0; u < UNR; ++u) v[u] = *reinterpret_cast<const uint4*>(sp[u]);
#pragma unroll
      for (int u = 0; u < UNR; ++u) {
        if (scale != 1.f) {
          __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&v[u]);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            float2 f = __bfloat1622float2(h[q]);
            h[q] = __floats2bfloat162_rn(f.x * scale, f.y * scale);
          }
        }
        if (ok[u]) *reinterpret_cast<uint4*>(dp[u]) = v[u];
      }
    } else {
      float4 v[UNR][VEC / 4];
#pragma unroll
      for (int u = 0; u < UNR; ++u)
#pragma unroll
        for (int q = 0; q < VEC / 4; ++q) v[u][q] = Vec4<S>::ld(sp[u] + 4 * q);
#pragma unroll
      for (int u = 0; u < UNR; ++u) {
        if (!ok[u]) continue;
#pragma unroll
        for (int q = 0; q < VEC / 4; ++q) Vec4<D>::st(dp[u] + 4 * q, scale != 1.f ? f4_scale(v[u][q], scale) : v[u][q]);
      }
    }
  }
}

TRB_API int trb_grad_push(const void* src, int s_dtype, int64_t src_stride, const int32_t* chunks, int n_chunks, int vec, void* const* dst_ptrs, int n_dst,
                          int d_dtype, int64_t dst_pitch, int64_t row_base, int B_local, float scale, cudaStream_t stream) {
  if (n_dst < 1 || n_dst > TRB_MAX_PEERS || (vec != 4 && vec != 8)) return -1;
  const int64_t n = (int64_t) B_local * n_chunks;
  if (n == 0) return 0;
  TrbPeerPtrs d;
  for (int i = 0; i < n_dst; ++i) d.p[i] = dst_ptrs[i];
  const int threads = 256;
  constexpr int UNR = 4;
  constexpr int kPushCtasPerSm = 2;  // persistent, but leaves room on every SM for the GEMMs that run beside the push
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  int64_t want = (n + (int64_t) threads * UNR - 1) / ((int64_t) threads * UNR);
  const unsigned blocks = (unsigned) (want < (int64_t) sms * kPushCtasPerSm ? want : (int64_t) sms * kPushCtasPerSm);
#define TRB_GP(SC, ST, DC, DT)                                                                                                                           \
  if (s_dtype == SC && d_dtype == DC) {                                                                                                                  \
    if (vec == 8) trb_grad_push_kernel<ST, DT, 8, UNR><<<blocks, threads, 0, stream>>>((const ST*) src, src_stride, chunks, n_chunks, d, dst_pitch, row_base, B_local, scale); \
    else trb_grad_push_kernel<ST, DT, 4, UNR><<<blocks, threads, 0, stream>>>((const ST*) src, src_stride, chunks, n_chunks, d, dst_pitch, row_base, B_local, scale);          \
    TRB_CHECK_LAUNCH();                                                                                                                                   \
    return 0;                                                                                                                                             \
  }
  TRB_GP(TRB_F32, float, TRB_F32, float)
  TRB_GP(TRB_F32, float, TRB_BF16, __nv_bfloat16)
  TRB_GP(TRB_BF16, __nv_bfloat16, TRB_F32, float)
  TRB_GP(TRB_BF16, __nv_bfloat16, TRB_BF16, __nv_bfloat16)
#undef TRB_GP
  return -3;
}

// ---------------------------------------------------------------------------------------------------------------
// FP8 wire of the sparse plane (format: qcomm_fp8.cuh). The push quantizes each gradient chunk of R = row_dim columns on the
// source and stores e4m3 payload + one fp32 scale into the owner's FP8 inbox; after the barrier `trb_fp8_wire_decode` turns
// payload + scales back into wire-dtype rows (the gradient inbox, or the pooled output of the forward).
// ---------------------------------------------------------------------------------------------------------------
// L = row_dim / 8 lanes per chunk, 8 values per lane; the lanes of a chunk are adjacent and aligned inside a warp, and since the
// work count is a multiple of L they enter and leave the grid-stride loop together (the amax shuffle needs all of them).
template <typename S, int UNR>
__global__ void __launch_bounds__(256)
trb_grad_push_fp8_kernel(const S* __restrict__ src, int64_t src_stride, const int32_t* __restrict__ chunks, int n_chunks, TrbPeerPtrs dst,
                         TrbPeerPtrs dst_scale, int64_t dst_pitch, int64_t scale_pitch, int64_t row_base, int B_local, int L) {
  const int64_t total = (int64_t) B_local * n_chunks * L;
  const int64_t stride = (int64_t) gridDim.x * blockDim.x;
  const int lane = threadIdx.x & 31;
  const unsigned gmask = L == 32 ? 0xffffffffu : ((1u << L) - 1u) << (lane & ~(L - 1));
  const int lig = lane & (L - 1);
  for (int64_t i0 = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i0 < total; i0 += stride * UNR) {
    float4 v[UNR][2];
    int64_t row[UNR];
    int rank[UNR], dc[UNR];
    bool ok[UNR];
#pragma unroll
    for (int u = 0; u < UNR; ++u) {
      const int64_t i = i0 + u * stride;
      ok[u] = i < total;
      const int64_t item = (ok[u] ? i : i0) / L;
      const int64_t b = item / n_chunks;
      const int c = (int) (item - b * n_chunks);
      rank[u] = chunks[3 * c];
      dc[u] = chunks[3 * c + 2];
      row[u] = row_base + b;
      const S* sp = src + b * src_stride + chunks[3 * c + 1] + lig * 8;
      v[u][0] = Vec4<S>::ld(sp);
      v[u][1] = Vec4<S>::ld(sp + 4);
    }
#pragma unroll
    for (int u = 0; u < UNR; ++u) {
      float amax = fmaxf(trb_fp8_abs_max4(v[u][0]), trb_fp8_abs_max4(v[u][1]));
      for (int o = L >> 1; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(gmask, amax, o));
      if (!ok[u]) continue;
      const float scale = trb_fp8_scale(amax);
      const float inv = 1.f / scale;
      uint8_t* q = reinterpret_cast<uint8_t*>(dst.p[rank[u]]) + row[u] * dst_pitch + dc[u] + lig * 8;
      *reinterpret_cast<uint2*>(q) = make_uint2(trb_fp8_encode4(v[u][0], inv), trb_fp8_encode4(v[u][1], inv));
      if (lig == 0) reinterpret_cast<float*>(dst_scale.p[rank[u]])[row[u] * scale_pitch + dc[u] / (8 * L)] = scale;
    }
  }
}

// chunks: int32 [n_chunks, 3] (destination rank, source column, inbox column), each `row_dim` (32 | 64 | 128) columns wide.
// dst_ptrs / scale_ptrs: every rank's uint8 payload inbox [*, dst_pitch] and fp32 scale inbox [*, scale_pitch]; source row b lands
// in row row_base + b.
TRB_API int trb_grad_push_fp8(const void* src, int s_dtype, int64_t src_stride, const int32_t* chunks, int n_chunks, int row_dim, void* const* dst_ptrs,
                              void* const* scale_ptrs, int n_dst, int64_t dst_pitch, int64_t scale_pitch, int64_t row_base, int B_local, cudaStream_t stream) {
  if (n_dst < 1 || n_dst > TRB_MAX_PEERS || (row_dim != 32 && row_dim != 64 && row_dim != 128)) return -1;
  const int L = row_dim / 8;
  const int64_t n = (int64_t) B_local * n_chunks * L;
  if (n == 0) return 0;
  TrbPeerPtrs d, ds;
  for (int i = 0; i < n_dst; ++i) {
    d.p[i] = dst_ptrs[i];
    ds.p[i] = scale_ptrs[i];
  }
  const int threads = 256;
  constexpr int UNR = 4;
  constexpr int kPushCtasPerSm = 2;  // as trb_grad_push: leaves room for the GEMMs that run beside the push
  const int sms = trb_num_sms();
  const int64_t want = (n + (int64_t) threads * UNR - 1) / ((int64_t) threads * UNR);
  const unsigned blocks = (unsigned) (want < (int64_t) sms * kPushCtasPerSm ? want : (int64_t) sms * kPushCtasPerSm);
  if (s_dtype == TRB_F32) {
    trb_grad_push_fp8_kernel<float, UNR><<<blocks, threads, 0, stream>>>((const float*) src, src_stride, chunks, n_chunks, d, ds, dst_pitch, scale_pitch, row_base, B_local, L);
  } else if (s_dtype == TRB_BF16) {
    trb_grad_push_fp8_kernel<__nv_bfloat16, UNR><<<blocks, threads, 0, stream>>>((const __nv_bfloat16*) src, src_stride, chunks, n_chunks, d, ds, dst_pitch, scale_pitch,
                                                                                 row_base, B_local, L);
  } else {
    return -3;
  }
  TRB_CHECK_LAUNCH();
  return 0;
}

// out[r, c : c + 16] = decode(payload[r, c : c + 16], scales[r, c / row_dim]) stored as O, for every row r < rows and every 16-column
// chunk start c in `cols` (a static list: the FP8 columns only, other columns of `out` are left alone). One 16-byte load per thread.
template <typename O>
__global__ void __launch_bounds__(256)
trb_fp8_wire_decode_kernel(const uint8_t* __restrict__ pay, int64_t pay_pitch, const float* __restrict__ scales, int64_t scale_pitch, int row_dim,
                           const int32_t* __restrict__ cols, int n_cols, int64_t rows, O* __restrict__ out, int64_t out_pitch) {
  const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * n_cols) return;
  const int64_t r = i / n_cols;
  const int c = cols[i - r * n_cols];
  const uint4 q = *reinterpret_cast<const uint4*>(pay + r * pay_pitch + c);
  const float s = scales[r * scale_pitch + c / row_dim];
  O* o = out + r * out_pitch + c;
  Vec4<O>::st(o, trb_fp8_decode4(q.x, s));
  Vec4<O>::st(o + 4, trb_fp8_decode4(q.y, s));
  Vec4<O>::st(o + 8, trb_fp8_decode4(q.z, s));
  Vec4<O>::st(o + 12, trb_fp8_decode4(q.w, s));
}

TRB_API int trb_fp8_wire_decode(const void* payload, int64_t pay_pitch, const float* scales, int64_t scale_pitch, int row_dim, const int32_t* cols, int n_cols,
                                int64_t rows, void* out, int out_dtype, int64_t out_pitch, cudaStream_t stream) {
  if (row_dim % 16 != 0 || pay_pitch % 16 != 0) return -1;
  const int64_t n = rows * n_cols;
  if (n == 0) return 0;
  const int threads = 256;
  const unsigned blocks = (unsigned) ((n + threads - 1) / threads);
  if (out_dtype == TRB_F32) {
    trb_fp8_wire_decode_kernel<float><<<blocks, threads, 0, stream>>>((const uint8_t*) payload, pay_pitch, scales, scale_pitch, row_dim, cols, n_cols, rows,
                                                                     (float*) out, out_pitch);
  } else if (out_dtype == TRB_BF16) {
    trb_fp8_wire_decode_kernel<__nv_bfloat16><<<blocks, threads, 0, stream>>>((const uint8_t*) payload, pay_pitch, scales, scale_pitch, row_dim, cols, n_cols,
                                                                             rows, (__nv_bfloat16*) out, out_pitch);
  } else {
    return -3;
  }
  TRB_CHECK_LAUNCH();
  return 0;
}
