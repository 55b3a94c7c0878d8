// DLRM dot-interaction forward / backward on wgmma tensor cores (sm_90a).
//
//   X_b = [dense_b ; sparse_b]            (R = F+1 rows, D columns, R <= 32, D == 128)
//   out_b = [dense_b , strict-upper-triangle(X_b X_b^T)]         (reference models/dlrm.py:210-222)
//
// The per-sample 27x27 products are far too small for a 64-row MMA, so FOUR samples are packed into
// one 128 x 128 operand tile (32 rows per sample, unused rows zero) in shared memory (SWIZZLE_128B).
// The CTA is one warpgroup; each 64-row half (two samples) is multiplied with itself by wgmma
// (m64n64k16, fp32 accumulators in registers) and only the two diagonal 32x32 blocks are kept.
// The 2x redundant FLOPs are free (the kernel is HBM-bound) and the operands never leave shared memory.
//
// Backward: dX_b = S_b X_b with S_b the symmetric 27x27 matrix rebuilt from the triangle of the
// incoming gradient. Tile math: D[128 x 128] = blockdiag(S)[128 x 128] . T[128 x 128] where the SAME
// shared-memory image of T (row-major, SWIZZLE_128B) is consumed as an MN-major B operand — no transpose.
//
// CTAs are small (128 threads, ~38 KB smem) so several fit per SM and hide the global load latency of
// each other; each CTA loops over groups of 4 samples.
#include "wgmma.cuh"

using namespace trb;

namespace {

constexpr int kD = 128;          // embedding dim handled by this kernel
constexpr int kRowsPerSample = 32;
constexpr int kSamples = 4;      // per MMA tile
constexpr int kTileBytes = 128 * 64 * 2;  // one [128 x 64] bf16 K-block

struct InterParams {
  const void* dense;     // [B, D] bf16
  int64_t ld_dense;
  const void* sparse;    // [B, F*D] (bf16 or fp32), row pitch ld_sparse
  int64_t ld_sparse;
  int sparse_f32;
  void* out;             // fwd: [B, ld_out] bf16
  int64_t ld_out;
  int B, F;
  int out_cols;          // D + R(R-1)/2
  // backward
  const void* gout;      // [B, ld_out] bf16
  void* g_dense;         // [B, D] bf16
  int64_t ld_gdense;
  void* g_sparse;        // [B, F*D] (bf16 or fp32)
  int64_t ld_gsparse;
  int gsparse_f32;
};

__device__ __forceinline__ int tri_offset(int i, int R) { return i * R - (i * (i + 1)) / 2; }  // first (i, i+1) slot

// Load the packed operand tile T (4 samples x 32 rows x 128 cols) into two SWIZZLE_128B K-blocks.
// Each thread moves 8 elements (16 B in smem). 128 threads: 4 samples x R rows x 16 chunks.
__device__ __forceinline__ void load_tile(const InterParams& p, uint8_t* tile, int b0, int tid) {
  const int R = p.F + 1;
  const int chunks = kSamples * R * 16;  // 16-byte chunks (8 bf16)
  for (int c = tid; c < chunks; c += 128) {
    const int s = c / (R * 16);
    const int rem = c - s * R * 16;
    const int i = rem >> 4;
    const int ch = rem & 15;  // chunk along D: columns [8*ch, 8*ch+8)
    const int b = b0 + s;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (b < p.B) {
      if (i == 0) {
        v = *reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(p.dense) + (int64_t) b * p.ld_dense + ch * 8);
      } else if (!p.sparse_f32) {
        v = *reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(p.sparse) + (int64_t) b * p.ld_sparse + (i - 1) * kD + ch * 8);
      } else {
        const float* src = reinterpret_cast<const float*>(p.sparse) + (int64_t) b * p.ld_sparse + (i - 1) * kD + ch * 8;
        const float4 f0 = *reinterpret_cast<const float4*>(src), f1 = *reinterpret_cast<const float4*>(src + 4);
        __nv_bfloat162 h0 = __floats2bfloat162_rn(f0.x, f0.y), h1 = __floats2bfloat162_rn(f0.z, f0.w);
        __nv_bfloat162 h2 = __floats2bfloat162_rn(f1.x, f1.y), h3 = __floats2bfloat162_rn(f1.z, f1.w);
        v.x = *reinterpret_cast<uint32_t*>(&h0); v.y = *reinterpret_cast<uint32_t*>(&h1);
        v.z = *reinterpret_cast<uint32_t*>(&h2); v.w = *reinterpret_cast<uint32_t*>(&h3);
      }
    }
    const int r = s * kRowsPerSample + i;
    const int kb = ch >> 3;  // which 64-column K-block
    const int k = (ch & 7) * 8;
    *reinterpret_cast<uint4*>(tile + kb * kTileBytes + sw128_offset(r, k)) = v;
  }
}

__device__ __forceinline__ void cp_async16(uint32_t smem_addr, const void* g, bool valid) {
  const int sz = valid ? 16 : 0;  // src-size 0 -> zero fill
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_addr), "l"(g), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// issue (do not wait for) the loads of the packed tile of samples [b0, b0+4): bf16 dense + bf16 sparse.
// Thread t always moves column chunk (t & 15) of rows (t >> 4) + 8k, so the swizzle term and all strides are per-thread
// constants (recomputing them per chunk made the kernel instruction-bound).
// EXTRA: also load gout[b][0:128] (the pass-through gradient of the dense row) as packed row R, so the backward MMA adds it
// in fp32 through S[0][R] = 1 instead of a lane-0 epilogue special case.
template <bool EXTRA>
__device__ __forceinline__ void issue_tile_loads(const InterParams& p, uint8_t* tile, int b0, int tid) {
  const int R = p.F + 1;
  const int ch = tid & 15, i0 = tid >> 4;
  const uint32_t tbase = smem_u32(tile) + (ch >> 3) * kTileBytes + ((((ch & 7) ^ (i0 & 7)) & 7) << 4);
  const __nv_bfloat16* dense = reinterpret_cast<const __nv_bfloat16*>(p.dense) + ch * 8;
  const __nv_bfloat16* sparse = reinterpret_cast<const __nv_bfloat16*>(p.sparse) + ch * 8 - kD;  // row i (>= 1) lives at + i * kD
  const __nv_bfloat16* gout = reinterpret_cast<const __nv_bfloat16*>(p.gout) + ch * 8;
#pragma unroll
  for (int s = 0; s < kSamples; ++s) {
    const int b = b0 + s;
    const bool ok = b < p.B;
    const int64_t bb = ok ? b : 0;
    const __nv_bfloat16* srow = sparse + bb * p.ld_sparse;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int i = i0 + 8 * k;
      const uint32_t dst = tbase + (uint32_t) ((s * kRowsPerSample + i) * 128);
      if (i < R) {
        cp_async16(dst, (i == 0) ? dense + bb * p.ld_dense : srow + (int64_t) i * kD, ok);
      } else if (EXTRA && i == R) {
        cp_async16(dst, gout + bb * p.ld_out, ok);
      }
    }
  }
}

// issue the loads of the 4 incoming-gradient rows (bwd)
__device__ __forceinline__ void issue_gout_loads(const InterParams& p, __nv_bfloat16* gstage, int b0, int tid) {
  const int vec_per_row = (int) (p.ld_out >> 3);
  const uint32_t gbase = smem_u32(gstage);
#pragma unroll
  for (int sidx = 0; sidx < kSamples; ++sidx) {
    const bool ok = b0 + sidx < p.B;
    const __nv_bfloat16* src = reinterpret_cast<const __nv_bfloat16*>(p.gout) + (int64_t) (ok ? b0 + sidx : 0) * p.ld_out;
    for (int c = tid; c < vec_per_row; c += 128) cp_async16(gbase + (uint32_t) (sidx * p.ld_out + c * 8) * 2, src + c * 8, ok);
  }
}

// ---- tensor-core pieces shared by the kernels (all 128 threads = one warpgroup; warp w, lane l) ----------------------
// Forward: Z = T T^T is only needed on the four diagonal 32 x 32 blocks. wgmma M-half h (packed rows [64h, 64h + 64) =
// samples 2h, 2h + 1) is multiplied with the same 64 rows only (N = 64): 2 x (m64n64k16 x 8) instead of a 128 x 128 product.
__device__ __forceinline__ void fwd_mma_issue(uint32_t tile_addr, float (&z)[2][32]) {
  wgmma_fence();
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int kb = 0; kb < 2; ++kb)
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint64_t desc = make_kmajor_desc(tile_addr + kb * kTileBytes + h * 8192 + k * 32);
        wgmma_m64n64k16<0, 0>(z[h], desc, desc, (kb | k) != 0);
      }
  wgmma_commit();
}

__device__ __forceinline__ void mma_wait(float (&z)[2][32]) {
  wgmma_wait<0>();
  wgmma_fence_regs(z[0]);
  wgmma_fence_regs(z[1]);
}

// strict upper triangle of the diagonal blocks -> the staged output rows (stage[s][kD + tri(i) + (j - i - 1)])
__device__ __forceinline__ void fwd_scatter(const float (&z)[2][32], __nv_bfloat16* stage, int64_t ld_out, int R, int warp, int lane) {
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int row = 16 * warp + (lane >> 2) + 8 * hh, col = 8 * j + 2 * (lane & 3) + c;  // inside M-half h
          const int i = row & 31, jj = col & 31;
          if ((row >> 5) == (col >> 5) && i < jj && jj < R)
            stage[(2 * h + (row >> 5)) * ld_out + kD + tri_offset(i, R) + (jj - i - 1)] = __float2bfloat16(z[h][4 * j + 2 * hh + c]);
        }
}

// Backward: D = blockdiag(S) . T. M-half h of blockdiag(S) is zero outside K-block h, so each half is 4 x m64n128k16 with
// A = S (K-major) and B = T consumed MN-major ([k = packed row][n = dim]; the two 64-column halves are kTileBytes apart).
// The halves run one after the other (64 accumulator registers instead of 128). Half h reads only rows [64h, 64h + 64) of K-block h
// of S, so the output of half 0 may already overwrite K-block 0 while half 1 runs.
__device__ __forceinline__ void bwd_mma_half(uint32_t aS, uint32_t aT, int h, float (&d)[64]) {
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const uint64_t adesc = make_kmajor_desc(aS + h * kTileBytes + h * 8192 + k * 32);
    const uint64_t bdesc = make_smem_desc(aT + (h * 64 + k * 16) * 128, kTileBytes, 1024);
    wgmma_m64n128k16<0, 1>(d, adesc, bdesc, k != 0);
  }
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_regs(d);
}

__global__ void __launch_bounds__(128, 4) interaction_fwd_kernel(const InterParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t) 1023);
  uint8_t* tile = smem;                                            // 2 x 16 KB
  __nv_bfloat16* stage = reinterpret_cast<__nv_bfloat16*>(smem + 2 * kTileBytes);  // [4][ld_out] output staging
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int R = p.F + 1;

  // zero the operand tile once: padding rows (i >= R) are never written again
  for (int i = tid; i < 2 * kTileBytes / 16; i += 128) reinterpret_cast<uint4*>(tile)[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  const int groups = (p.B + kSamples - 1) / kSamples;
  for (int g = blockIdx.x; g < groups; g += gridDim.x) {
    const int b0 = g * kSamples;
    load_tile(p, tile, b0, tid);
    fence_proxy_async();  // generic-proxy smem writes -> visible to the tensor-core (async) proxy
    __syncthreads();
    float z[2][32];
    fwd_mma_issue(smem_u32(tile), z);
    mma_wait(z);
    fwd_scatter(z, stage, p.ld_out, R, warp, lane);
    // dense passthrough + zero padding of the row tail (warp w <-> sample b0 + w)
    __nv_bfloat16* srow = stage + warp * p.ld_out;
    for (int c = lane; c < kD / 8; c += 32) {
      const int r = warp * kRowsPerSample;
      reinterpret_cast<uint4*>(srow)[c] = *reinterpret_cast<const uint4*>(tile + (c >> 3) * kTileBytes + sw128_offset(r, (c & 7) * 8));
    }
    for (int c = p.out_cols + lane; c < p.ld_out; c += 32) srow[c] = __float2bfloat16(0.f);
    __syncthreads();  // staging complete; operand tile free for the next group
    const int vec_per_row = (int) (p.ld_out >> 3);
    for (int v = tid; v < kSamples * vec_per_row; v += 128) {
      const int s = v / vec_per_row, c = v - s * vec_per_row;
      if (b0 + s < p.B)
        reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.out) + (int64_t) (b0 + s) * p.ld_out)[c] =
            reinterpret_cast<const uint4*>(stage + s * p.ld_out)[c];
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(128, 3) interaction_bwd_kernel(const InterParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t) 1023);
  uint8_t* tileT = smem;                     // packed X (2 K-blocks), used as MN-major B operand
  uint8_t* tileS = smem + 2 * kTileBytes;    // block-diagonal S (2 K-blocks), K-major A operand
  __nv_bfloat16* gstage = reinterpret_cast<__nv_bfloat16*>(smem + 4 * kTileBytes);  // [4][ld_out] incoming gradient rows
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int R = p.F + 1;

  for (int i = tid; i < 4 * kTileBytes / 16; i += 128) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  const int groups = (p.B + kSamples - 1) / kSamples;
  for (int g = blockIdx.x; g < groups; g += gridDim.x) {
    const int b0 = g * kSamples;
    load_tile(p, tileT, b0, tid);
    // stage the 4 incoming gradient rows with coalesced 16 B loads
    {
      const int vec_per_row = (int) (p.ld_out >> 3);
      for (int v = tid; v < kSamples * vec_per_row; v += 128) {
        const int sidx = v / vec_per_row, c = v - sidx * vec_per_row;
        uint4 val = make_uint4(0, 0, 0, 0);
        if (b0 + sidx < p.B) val = reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(p.gout) + (int64_t) (b0 + sidx) * p.ld_out)[c];
        reinterpret_cast<uint4*>(gstage + sidx * p.ld_out)[c] = val;
      }
    }
    __syncthreads();
    // S rows: thread (warp = sample, lane = i) writes S[i][j] for all j (symmetric, zero diagonal)
    {
      const int b = b0 + warp;
      const int r = warp * kRowsPerSample + lane;
      const __nv_bfloat16* grow = gstage + warp * p.ld_out + kD;
      if (lane < R) {
        for (int j = 0; j < R; ++j) {
          __nv_bfloat16 v = __float2bfloat16(0.f);
          if (b < p.B && j != lane) {
            const int lo = min(lane, j), hi = max(lane, j);
            v = grow[tri_offset(lo, R) + (hi - lo - 1)];
          }
          const int k = warp * kRowsPerSample + j;
          *reinterpret_cast<__nv_bfloat16*>(tileS + (k >> 6) * kTileBytes + sw128_offset(r, k & 63)) = v;
        }
      }
    }
    fence_proxy_async();
    __syncthreads();
    const int q = lane & 3;
#pragma unroll 1
    for (int h = 0; h < 2; ++h) {
      float d[64];
      bwd_mma_half(smem_u32(tileS), smem_u32(tileT), h, d);
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int r = 64 * h + 16 * warp + (lane >> 2) + 8 * hh;
        const int s = r >> 5, i = r & 31, b = b0 + s;
        if (b >= p.B || i >= R) continue;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int col = 8 * j + 2 * q;
          float v0 = d[4 * j + 2 * hh], v1 = d[4 * j + 2 * hh + 1];
          if (i == 0) {
            // dense row: add the pass-through gradient of out[:, :D]
            const __nv_bfloat162 gd = *reinterpret_cast<const __nv_bfloat162*>(gstage + s * p.ld_out + col);
            v0 += __bfloat162float(gd.x);
            v1 += __bfloat162float(gd.y);
            *reinterpret_cast<__nv_bfloat162*>(reinterpret_cast<__nv_bfloat16*>(p.g_dense) + (int64_t) b * p.ld_gdense + col) = __floats2bfloat162_rn(v0, v1);
          } else if (p.gsparse_f32) {
            *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.g_sparse) + (int64_t) b * p.ld_gsparse + (i - 1) * kD + col) = make_float2(v0, v1);
          } else {
            *reinterpret_cast<__nv_bfloat162*>(reinterpret_cast<__nv_bfloat16*>(p.g_sparse) + (int64_t) b * p.ld_gsparse + (i - 1) * kD + col) =
                __floats2bfloat162_rn(v0, v1);
          }
        }
      }
    }
    __syncthreads();
  }
}


// ================================================================================================================
// Pipelined bf16 kernels (the production path): operand tiles arrive through cp.async (16 B LDGSTS, every thread has
// all of its loads in flight at once) into a DOUBLE-BUFFERED smem image, so the global->smem traffic of group g+1
// overlaps the MMA + epilogue of group g; results leave through a swizzled smem staging area with fully coalesced
// 16 B stores. The kernels above (synchronous loads, per-thread 4 B stores) remain as the fp32-I/O fallback.
// ================================================================================================================

__global__ void __launch_bounds__(128, 3) interaction_fwd_pipe_kernel(const InterParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t) 1023);
  uint8_t* tiles = smem;                                                               // 2 buffers x (2 x 16 KB)
  __nv_bfloat16* stage = reinterpret_cast<__nv_bfloat16*>(smem + 4 * kTileBytes);      // [4][ld_out]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int R = p.F + 1;
  for (int i = tid; i < 4 * kTileBytes / 16; i += 128) reinterpret_cast<uint4*>(tiles)[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  const int groups = (p.B + kSamples - 1) / kSamples;
  int cur = 0;
  if ((int) blockIdx.x < groups) issue_tile_loads<false>(p, tiles, blockIdx.x * kSamples, tid);
  cp_async_commit();
  for (int g = blockIdx.x; g < groups; g += gridDim.x, cur ^= 1) {
    const int b0 = g * kSamples;
    uint8_t* tile = tiles + cur * 2 * kTileBytes;
    cp_async_wait_all();
    fence_proxy_async();
    __syncthreads();  // tile[cur] landed; everyone is done with tile[cur^1] and with `stage`
    if (g + (int) gridDim.x < groups) issue_tile_loads<false>(p, tiles + (cur ^ 1) * 2 * kTileBytes, (g + gridDim.x) * kSamples, tid);
    cp_async_commit();
    float z[2][32];
    fwd_mma_issue(smem_u32(tile), z);
    // dense passthrough + zero tail while the MMA runs
    __nv_bfloat16* srow = stage + warp * p.ld_out;
    for (int c = lane; c < kD / 8; c += 32) {
      const int r = warp * kRowsPerSample;
      reinterpret_cast<uint4*>(srow)[c] = *reinterpret_cast<const uint4*>(tile + (c >> 3) * kTileBytes + sw128_offset(r, (c & 7) * 8));
    }
    for (int c = p.out_cols + lane; c < p.ld_out; c += 32) srow[c] = __float2bfloat16(0.f);
    mma_wait(z);
    fwd_scatter(z, stage, p.ld_out, R, warp, lane);
    __syncthreads();
    const int vec_per_row = (int) (p.ld_out >> 3);
#pragma unroll
    for (int s = 0; s < kSamples; ++s) {
      if (b0 + s >= p.B) break;
      uint4* orow = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.out) + (int64_t) (b0 + s) * p.ld_out);
      const uint4* srow4 = reinterpret_cast<const uint4*>(stage + s * p.ld_out);
      for (int c = tid; c < vec_per_row; c += 128) orow[c] = srow4[c];
    }
  }
  cp_async_wait_all();
}

template <bool EXTRA>
__global__ void __launch_bounds__(128, 2) interaction_bwd_pipe_kernel(const InterParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t) 1023);
  uint8_t* tiles = smem;                       // T: 2 buffers x 32 KB (MN-major B operand)
  uint8_t* tileS = smem + 4 * kTileBytes;      // S (K-major A operand, 32 KB); re-used as the output staging area after the MMA
  __nv_bfloat16* gst = reinterpret_cast<__nv_bfloat16*>(smem + 6 * kTileBytes);  // 2 x [4][ld_out]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int R = p.F + 1;
  for (int i = tid; i < 4 * kTileBytes / 16; i += 128) reinterpret_cast<uint4*>(tiles)[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  const int groups = (p.B + kSamples - 1) / kSamples;
  const int gsz = kSamples * (int) p.ld_out;
  int cur = 0;
  if ((int) blockIdx.x < groups) {
    issue_tile_loads<EXTRA>(p, tiles, blockIdx.x * kSamples, tid);
    issue_gout_loads(p, gst, blockIdx.x * kSamples, tid);
  }
  cp_async_commit();
  const int r = warp * kRowsPerSample + lane;  // my row of the packed tile (sample = warp, row-in-sample = lane)
  for (int g = blockIdx.x; g < groups; g += gridDim.x, cur ^= 1) {
    const int b0 = g * kSamples;
    uint8_t* tileT = tiles + cur * 2 * kTileBytes;
    const __nv_bfloat16* gstage = gst + cur * gsz;
    cp_async_wait_all();
    fence_proxy_async();
    __syncthreads();  // T[cur] / gout[cur] landed; copy-out of the previous group finished (staging == tileS is free)
    if (g + (int) gridDim.x < groups) {
      issue_tile_loads<EXTRA>(p, tiles + (cur ^ 1) * 2 * kTileBytes, (g + gridDim.x) * kSamples, tid);
      issue_gout_loads(p, gst + (cur ^ 1) * gsz, (g + gridDim.x) * kSamples, tid);
    }
    cp_async_commit();
    // ---- S row of this thread: S[i][j] = g[triangle(min,max)] (0 on the diagonal / padding); the whole 256 B row of
    //      blockdiag(S) is written (zeros outside the sample's own 32-column block) because the staging re-use clobbers it
    {
      const __nv_bfloat16* grow = gstage + warp * p.ld_out + kD;
      const bool live = lane < R && (b0 + warp) < p.B;
      // S[i][j] = g[tri(min) + (max - min - 1)]: for j < i the offset walks down the column (stride R - j - 2), for j > i it
      // is contiguous in the row of i — no multiplications inside the loop
      uint32_t packed[16];
      int off_lo = lane - 1;
      const int off_hi = tri_offset(lane, R) - (lane + 1);
#pragma unroll
      for (int j2 = 0; j2 < 16; ++j2) {
        __nv_bfloat16 v[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int j = 2 * j2 + h;
          v[h] = __float2bfloat16(0.f);
          if (live && j < R && j != lane) v[h] = grow[(j < lane) ? off_lo : off_hi + j];
          if (EXTRA && j == R && lane == 0) v[h] = __float2bfloat16(1.f);  // routes packed row R (pass-through gradient) into the dense row
          off_lo += R - j - 2;
        }
        __nv_bfloat162 hh = __halves2bfloat162(v[0], v[1]);
        packed[j2] = *reinterpret_cast<uint32_t*>(&hh);
      }
      // row r: K-block kb holds k in [64 kb, 64 kb + 64) as 8 chunks of 16 B; own block = k in [32 warp, 32 warp + 32)
      const int own_kb = warp >> 1, own_c0 = (warp & 1) * 4;
#pragma unroll
      for (int kb = 0; kb < 2; ++kb) {
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          uint4 val = make_uint4(0, 0, 0, 0);
          if (kb == own_kb && c >= own_c0 && c < own_c0 + 4) {
            const int q = (c - own_c0) * 4;
            val = make_uint4(packed[q], packed[q + 1], packed[q + 2], packed[q + 3]);
          }
          *reinterpret_cast<uint4*>(tileS + kb * kTileBytes + r * 128 + (((c ^ (r & 7)) & 7) << 4)) = val;
        }
      }
    }
    fence_proxy_async();
    __syncthreads();
    // ---- per half: MMA, then registers -> bf16 -> swizzled staging ([128 rows][16 chunks of 16 B], chunk ^= row & 15). The
    //      staging rows of half h are K-block h of S, which only half h reads: its wgmma has retired when the stores start.
    uint8_t* ostage = tileS;
    const int q = lane & 3;
#pragma unroll 1
    for (int h = 0; h < 2; ++h) {
      float d[64];
      bwd_mma_half(smem_u32(tileS), smem_u32(tileT), h, d);
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int rr = 64 * h + 16 * warp + (lane >> 2) + 8 * hh;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          float v0 = d[4 * j + 2 * hh], v1 = d[4 * j + 2 * hh + 1];
          if (!EXTRA && (rr & 31) == 0) {  // R == 32: no spare packed row, add the pass-through gradient of out[:, :D] here
            const __nv_bfloat162 gd = *reinterpret_cast<const __nv_bfloat162*>(gstage + (rr >> 5) * p.ld_out + 8 * j + 2 * q);
            v0 += __bfloat162float(gd.x);
            v1 += __bfloat162float(gd.y);
          }
          *reinterpret_cast<__nv_bfloat162*>(ostage + rr * 256 + (((j ^ rr) & 15) << 4) + 4 * q) = __floats2bfloat162_rn(v0, v1);
        }
      }
    }
    __syncthreads();
    // ---- coalesced copy-out: 16 consecutive threads write one 256 B gradient row; thread t owns chunk (t & 15) of rows (t >> 4) + 8k
    {
      const int ch = tid & 15, i0 = tid >> 4;
      __nv_bfloat16* gd_base = reinterpret_cast<__nv_bfloat16*>(p.g_dense) + ch * 8;
      __nv_bfloat16* gs_base = reinterpret_cast<__nv_bfloat16*>(p.g_sparse) + ch * 8 - kD;
#pragma unroll
      for (int s4 = 0; s4 < kSamples; ++s4) {
        const int b = b0 + s4;
        if (b >= p.B) break;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int i = i0 + 8 * k;
          if (i >= R) break;
          const uint4 val = *reinterpret_cast<const uint4*>(ostage + (s4 * kRowsPerSample + i) * 256 + (((ch ^ i) & 15) << 4));
          __nv_bfloat16* dst = (i == 0) ? gd_base + (int64_t) b * p.ld_gdense : gs_base + (int64_t) b * p.ld_gsparse + (int64_t) i * kD;
          *reinterpret_cast<uint4*>(dst) = val;
        }
      }
    }
  }
  cp_async_wait_all();
}

int g_sms = 0;
int num_sms() {
  if (g_sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, dev);
  }
  return g_sms;
}

}  // namespace

// out[b] = [dense_b, triu(X_b X_b^T, 1)] with ld_out >= D + R(R-1)/2 (multiple of 8, tail zero filled)
TRB_API int trb_interaction_fwd(const void* dense, int64_t ld_dense, const void* sparse, int64_t ld_sparse, int sparse_f32, void* out,
                                int64_t ld_out, int B, int F, int D, cudaStream_t stream) {
  if (D != kD || F + 1 > 32 || F < 1) return -20;
  if (B == 0) return 0;
  InterParams p = {};
  p.dense = dense; p.ld_dense = ld_dense; p.sparse = sparse; p.ld_sparse = ld_sparse; p.sparse_f32 = sparse_f32;
  p.out = out; p.ld_out = ld_out; p.B = B; p.F = F; p.out_cols = D + (F + 1) * F / 2;
  if (ld_out % 8 || ld_out < p.out_cols) return -21;
  const int groups = (B + kSamples - 1) / kSamples;
  if (!sparse_f32 && ld_dense % 8 == 0 && ld_sparse % 8 == 0) {
    const int smem_p = 4 * kTileBytes + kSamples * (int) ld_out * 2 + 64 + 1024;
    static bool cfg_p = false;
    if (!cfg_p) {
      TRB_CUDA(cudaFuncSetAttribute(interaction_fwd_pipe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
      cfg_p = true;
    }
    const int grid_p = groups < 3 * num_sms() ? groups : 3 * num_sms();
    interaction_fwd_pipe_kernel<<<grid_p, 128, smem_p, stream>>>(p);
    TRB_CHECK_LAUNCH();
    return 0;
  }
  const int smem = 2 * kTileBytes + kSamples * (int) ld_out * 2 + 64 + 1024;
  static bool cfg = false;
  if (!cfg) {
    TRB_CUDA(cudaFuncSetAttribute(interaction_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    cfg = true;
  }
  const int grid = groups < 4 * num_sms() ? groups : 4 * num_sms();
  interaction_fwd_kernel<<<grid, 128, smem, stream>>>(p);
  TRB_CHECK_LAUNCH();
  return 0;
}

TRB_API int trb_interaction_bwd(const void* dense, int64_t ld_dense, const void* sparse, int64_t ld_sparse, int sparse_f32, const void* gout,
                                int64_t ld_out, void* g_dense, int64_t ld_gdense, void* g_sparse, int64_t ld_gsparse, int gsparse_f32, int B,
                                int F, int D, cudaStream_t stream) {
  if (D != kD || F + 1 > 32 || F < 1) return -20;
  if (B == 0) return 0;
  InterParams p = {};
  p.dense = dense; p.ld_dense = ld_dense; p.sparse = sparse; p.ld_sparse = ld_sparse; p.sparse_f32 = sparse_f32;
  p.gout = gout; p.ld_out = ld_out; p.B = B; p.F = F; p.out_cols = D + (F + 1) * F / 2;
  p.g_dense = g_dense; p.ld_gdense = ld_gdense; p.g_sparse = g_sparse; p.ld_gsparse = ld_gsparse; p.gsparse_f32 = gsparse_f32;
  const int groups = (B + kSamples - 1) / kSamples;
  if (!sparse_f32 && !gsparse_f32 && ld_dense % 8 == 0 && ld_sparse % 8 == 0 && ld_gdense % 8 == 0 && ld_gsparse % 8 == 0 && ld_out % 8 == 0) {
    const int smem_p = 6 * kTileBytes + 2 * kSamples * (int) ld_out * 2 + 64 + 1024;
    static bool cfg_p = false;
    if (!cfg_p) {
      TRB_CUDA(cudaFuncSetAttribute(interaction_bwd_pipe_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024));
      TRB_CUDA(cudaFuncSetAttribute(interaction_bwd_pipe_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024));
      cfg_p = true;
    }
    const int grid_p = groups < 2 * num_sms() ? groups : 2 * num_sms();
    if (F + 1 < 32) interaction_bwd_pipe_kernel<true><<<grid_p, 128, smem_p, stream>>>(p);
    else interaction_bwd_pipe_kernel<false><<<grid_p, 128, smem_p, stream>>>(p);
    TRB_CHECK_LAUNCH();
    return 0;
  }
  const int smem = 4 * kTileBytes + kSamples * (int) ld_out * 2 + 64 + 1024;
  static bool cfg = false;
  if (!cfg) {
    TRB_CUDA(cudaFuncSetAttribute(interaction_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    cfg = true;
  }
  const int grid = groups < 3 * num_sms() ? groups : 3 * num_sms();
  interaction_bwd_kernel<<<grid, 128, smem, stream>>>(p);
  TRB_CHECK_LAUNCH();
  return 0;
}
