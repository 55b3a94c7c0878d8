// DLRM dot-interaction forward / backward on wgmma tensor cores (sm_90a): kernel templates over the embedding width D and the
// packing RPS (packed tile rows given to one sample). interaction.cu holds the C ABI and the D = 80 ... 128 instances; the other
// widths are instantiated in interaction_d*.cu so that the instances compile in parallel.
//
//   X_b = [dense_b ; sparse_b]            (R = F+1 rows, D columns; R <= RPS, 16 <= D <= 256, D % 16 == 0)
//   out_b = [dense_b , strict-upper-triangle(X_b X_b^T)]         (reference models/dlrm.py:210-222)
//
// The per-sample R x R products are far too small for a 64-row MMA, so 128 / RPS samples are packed into one 128-row operand
// tile (RPS rows per sample, unused rows zero) in shared memory: ceil(D / 64) SWIZZLE_128B K-blocks of [128 x 64] bf16, columns
// past D zero. RPS is the smallest of 16, 32, 64, 128 that holds R rows.
// The CTA is one warpgroup. For RPS <= 64 each 64-row half (64 / RPS samples) is multiplied with itself by wgmma (m64n64k16,
// D / 16 k-steps, fp32 accumulators in registers) and only the diagonal RPS x RPS blocks are kept; for RPS = 128 each half is
// multiplied with the whole tile (m64n128k16). The redundant FLOPs are free (the kernel is HBM-bound) and the operands never
// leave shared memory.
//
// Backward: dX_b = S_b X_b with S_b the symmetric R x R matrix rebuilt from the triangle of the incoming gradient. Tile math:
// D[128 x D] = blockdiag(S)[128 x 128] . T[128 x D] where the SAME shared-memory image of T (row-major, SWIZZLE_128B) is consumed
// as an MN-major B operand - no transpose. N is split into chunks of 128 columns (m64n128k16; m64n64k16 for an odd last K-block),
// so the accumulators stay at 64 registers per thread for every D.
//
// CTAs are small (128 threads) so several fit per SM and hide the global load latency of each other; each CTA loops over
// groups of 128 / RPS samples.
#pragma once
#include "wgmma.cuh"

namespace trb {

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

// launchers of one group of widths (interaction.cu, interaction_d*.cu); -20 for a width outside the group
int interaction_fwd_d16_64(const InterParams& p, int D, cudaStream_t stream);
int interaction_bwd_d16_64(const InterParams& p, int D, cudaStream_t stream);
int interaction_fwd_d80_128(const InterParams& p, int D, cudaStream_t stream);
int interaction_bwd_d80_128(const InterParams& p, int D, cudaStream_t stream);
int interaction_fwd_d144_192(const InterParams& p, int D, cudaStream_t stream);
int interaction_bwd_d144_192(const InterParams& p, int D, cudaStream_t stream);
int interaction_fwd_d208_256(const InterParams& p, int D, cudaStream_t stream);
int interaction_bwd_d208_256(const InterParams& p, int D, cudaStream_t stream);

}  // namespace trb

namespace {

using namespace trb;

constexpr int kTileBytes = 128 * 64 * 2;  // one [128 x 64] bf16 K-block

constexpr int ilog2(int x) { return x <= 1 ? 0 : 1 + ilog2(x >> 1); }

// Compile-time shape of one (D, RPS) instance.
template <int D, int RPS>
struct Shape {
  static_assert(D % 16 == 0 && D >= 16 && D <= 256, "D");
  static_assert(RPS == 16 || RPS == 32 || RPS == 64 || RPS == 128, "RPS");
  static constexpr int KB = (D + 63) / 64;           // SWIZZLE_128B K-blocks of the operand tile
  static constexpr int S = 128 / RPS;                // samples per tile
  static constexpr int CPR = D / 8;                  // 16-byte chunks per row
  static constexpr int LCPR = ilog2(CPR);            // log2(CPR) when CPR is a power of two
  static constexpr int LRPS = ilog2(RPS);
  static constexpr int SPH = RPS <= 64 ? 64 / RPS : 1;  // samples per 64-row M-half
  static constexpr int LSPH = ilog2(SPH);
  static constexpr int NF = RPS <= 64 ? 64 : 128;       // forward MMA width: the half itself, or the whole tile
  // thread t moves chunk (t % CPR) of the rows (t / CPR) + RSTEP k when CPR divides 128 and a sample spans RSTEP rows or more
  static constexpr bool kFixedChunk = (128 % CPR) == 0 && (128 / CPR) <= RPS;
  static constexpr int RSTEP = (128 % CPR) == 0 ? 128 / CPR : 1;
  // the pipelined backward stages its bf16 output in the S tile when the output fits in the rows of S its own M-half read
  static constexpr bool kStageInS = KB <= 2 && RPS <= 64;
  static constexpr int kMaxLdOut = (D + RPS * (RPS - 1) / 2 + 7) / 8 * 8;
  // CTAs per SM that the shared memory of the widest output row of this packing allows, at most `cap` (the register budget of
  // __launch_bounds__); a CTA needs `fixed` bytes plus `rows` staged output rows
  static constexpr int ctas(int cap, int fixed, int rows) {
    const int n = 233472 / (fixed + rows * kMaxLdOut * 2 + 64 + 2048);
    return n < 1 ? 1 : (n < cap ? n : cap);
  }
  static constexpr int kFwdCtas = ctas(RPS == 128 ? 2 : 4, KB * kTileBytes, S);
  static constexpr int kFwdPipeCtas = ctas(RPS == 128 ? 2 : 3, 2 * KB * kTileBytes, S);
  static constexpr int kBwdCtas = ctas(3, (KB + 2) * kTileBytes, S);
  static constexpr int kBwdPipeCtas = ctas(2, (2 * KB + 2) * kTileBytes, 2 * S);
};

__device__ __forceinline__ int tri_offset(int i, int R) { return i * R - (i * (i + 1)) / 2; }  // first (i, i+1) slot

// Load the packed operand tile T (S samples x RPS rows x D cols) into KB SWIZZLE_128B K-blocks.
// Each thread moves 8 elements (16 B in smem). 128 threads: S samples x R rows x CPR chunks.
template <int D, int RPS>
__device__ __forceinline__ void load_tile(const InterParams& p, uint8_t* tile, int b0, int tid) {
  using Sh = Shape<D, RPS>;
  const int R = p.F + 1;
  const int chunks = Sh::S * R * Sh::CPR;  // 16-byte chunks (8 bf16)
  for (int c = tid; c < chunks; c += 128) {
    const int s = c / (R * Sh::CPR);
    const int rem = c - s * R * Sh::CPR;
    const int i = (int) ((unsigned) rem / Sh::CPR);
    const int ch = (int) ((unsigned) rem % Sh::CPR);  // chunk along D: columns [8*ch, 8*ch+8)
    const int b = b0 + s;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (b < p.B) {
      if (i == 0) {
        v = *reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(p.dense) + (int64_t) b * p.ld_dense + ch * 8);
      } else if (!p.sparse_f32) {
        v = *reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(p.sparse) + (int64_t) b * p.ld_sparse + (i - 1) * D + ch * 8);
      } else {
        const float* src = reinterpret_cast<const float*>(p.sparse) + (int64_t) b * p.ld_sparse + (i - 1) * D + ch * 8;
        const float4 f0 = *reinterpret_cast<const float4*>(src), f1 = *reinterpret_cast<const float4*>(src + 4);
        __nv_bfloat162 h0 = __floats2bfloat162_rn(f0.x, f0.y), h1 = __floats2bfloat162_rn(f0.z, f0.w);
        __nv_bfloat162 h2 = __floats2bfloat162_rn(f1.x, f1.y), h3 = __floats2bfloat162_rn(f1.z, f1.w);
        v.x = *reinterpret_cast<uint32_t*>(&h0); v.y = *reinterpret_cast<uint32_t*>(&h1);
        v.z = *reinterpret_cast<uint32_t*>(&h2); v.w = *reinterpret_cast<uint32_t*>(&h3);
      }
    }
    const int r = s * RPS + i;
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

// issue (do not wait for) the loads of the packed tile of samples [b0, b0+S): bf16 dense + bf16 sparse.
// kFixedChunk: thread t always moves column chunk (t % CPR) of rows (t / CPR) + RSTEP k, so the swizzle term and all strides are
// per-thread constants (recomputing them per chunk made the kernel instruction-bound). Other widths walk the chunks of the tile.
// EXTRA: also load gout[b][0:D] (the pass-through gradient of the dense row) as packed row R, so the backward MMA adds it
// in fp32 through S[0][R] = 1 instead of a lane-0 epilogue special case.
template <int D, int RPS, bool EXTRA>
__device__ __forceinline__ void issue_tile_loads(const InterParams& p, uint8_t* tile, int b0, int tid) {
  using Sh = Shape<D, RPS>;
  const int R = p.F + 1;
  if constexpr (Sh::kFixedChunk) {
    constexpr int RSTEP = Sh::RSTEP;
    const int ch = tid & (Sh::CPR - 1), i0 = tid >> Sh::LCPR;
    const uint32_t kbase = smem_u32(tile) + (ch >> 3) * kTileBytes;
    const uint32_t tbase = kbase + ((((ch & 7) ^ (i0 & 7)) & 7) << 4);  // the swizzle term when RSTEP % 8 == 0
    const __nv_bfloat16* dense = reinterpret_cast<const __nv_bfloat16*>(p.dense) + ch * 8;
    const __nv_bfloat16* sparse = reinterpret_cast<const __nv_bfloat16*>(p.sparse) + ch * 8 - D;  // row i (>= 1) lives at + i * D
    const __nv_bfloat16* gout = reinterpret_cast<const __nv_bfloat16*>(p.gout) + ch * 8;
#pragma unroll
    for (int s = 0; s < Sh::S; ++s) {
      const int b = b0 + s;
      const bool ok = b < p.B;
      const int64_t bb = ok ? b : 0;
      const __nv_bfloat16* srow = sparse + bb * p.ld_sparse;
#pragma unroll
      for (int k = 0; k < RPS / RSTEP; ++k) {
        const int i = i0 + RSTEP * k;
        const int r = s * RPS + i;
        const uint32_t dst = (RSTEP % 8 == 0) ? tbase + (uint32_t) (r * 128) : kbase + (uint32_t) (r * 128) + ((((ch & 7) ^ (r & 7)) & 7) << 4);
        if (i < R) {
          cp_async16(dst, (i == 0) ? dense + bb * p.ld_dense : srow + (int64_t) i * D, ok);
        } else if (EXTRA && i == R) {
          cp_async16(dst, gout + bb * p.ld_out, ok);
        }
      }
    }
  } else {
    const uint32_t base = smem_u32(tile);
#pragma unroll
    for (int k = 0; k < Sh::CPR; ++k) {
      const int c = tid + 128 * k;
      const int r = (int) ((unsigned) c / Sh::CPR), ch = (int) ((unsigned) c % Sh::CPR);
      const int s = r >> Sh::LRPS, i = r & (RPS - 1);
      if (i > R || (!EXTRA && i == R)) continue;
      const int b = b0 + s;
      const bool ok = b < p.B;
      const int64_t bb = ok ? b : 0;
      const __nv_bfloat16* src = (i == 0) ? reinterpret_cast<const __nv_bfloat16*>(p.dense) + bb * p.ld_dense
                                 : (i < R) ? reinterpret_cast<const __nv_bfloat16*>(p.sparse) + bb * p.ld_sparse + (int64_t) (i - 1) * D
                                           : reinterpret_cast<const __nv_bfloat16*>(p.gout) + bb * p.ld_out;
      cp_async16(base + (ch >> 3) * kTileBytes + sw128_offset(r, (ch & 7) * 8), src + ch * 8, ok);
    }
  }
}

// issue the loads of the S incoming-gradient rows (bwd)
template <int S>
__device__ __forceinline__ void issue_gout_loads(const InterParams& p, __nv_bfloat16* gstage, int b0, int tid) {
  const int vec_per_row = (int) (p.ld_out >> 3);
  const uint32_t gbase = smem_u32(gstage);
#pragma unroll
  for (int sidx = 0; sidx < S; ++sidx) {
    const bool ok = b0 + sidx < p.B;
    const __nv_bfloat16* src = reinterpret_cast<const __nv_bfloat16*>(p.gout) + (int64_t) (ok ? b0 + sidx : 0) * p.ld_out;
    for (int c = tid; c < vec_per_row; c += 128) cp_async16(gbase + (uint32_t) (sidx * p.ld_out + c * 8) * 2, src + c * 8, ok);
  }
}

// ---- tensor-core pieces shared by the kernels (all 128 threads = one warpgroup; warp w, lane l) ----------------------
// Forward: Z = T T^T is only needed on the diagonal RPS x RPS blocks. For RPS <= 64, wgmma M-half h (packed rows
// [64h, 64h + 64)) is multiplied with the same 64 rows only (N = 64): 2 x (m64n64k16 x D/16) instead of a 128 x 128 product.
// For RPS = 128 the one sample spans both halves, and each half is multiplied with all 128 rows (N = 128).
template <int D, int RPS>
__device__ __forceinline__ void fwd_mma_issue(uint32_t tile_addr, float (&z)[2][Shape<D, RPS>::NF / 2]) {
  constexpr int KB = Shape<D, RPS>::KB;
  wgmma_fence();
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int kb = 0; kb < KB; ++kb)
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (kb * 4 + k >= D / 16) continue;
        const uint64_t desc = make_kmajor_desc(tile_addr + kb * kTileBytes + h * 8192 + k * 32);
        if constexpr (RPS <= 64) {
          wgmma_m64n64k16<0, 0>(z[h], desc, desc, (kb | k) != 0);
        } else {
          wgmma_m64n128k16<0, 0>(z[h], desc, make_kmajor_desc(tile_addr + kb * kTileBytes + k * 32), (kb | k) != 0);
        }
      }
  wgmma_commit();
}

template <int N>
__device__ __forceinline__ void mma_wait(float (&z)[2][N]) {
  wgmma_wait<0>();
  wgmma_fence_regs(z[0]);
  wgmma_fence_regs(z[1]);
}

// strict upper triangle of the diagonal blocks -> the staged output rows (stage[s][D + tri(i) + (j - i - 1)])
template <int D, int RPS>
__device__ __forceinline__ void fwd_scatter(const float (&z)[2][Shape<D, RPS>::NF / 2], __nv_bfloat16* stage, int64_t ld_out, int R, int warp,
                                            int lane) {
  using Sh = Shape<D, RPS>;
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int j = 0; j < Sh::NF / 8; ++j)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int row = 16 * warp + (lane >> 2) + 8 * hh, col = 8 * j + 2 * (lane & 3) + c;  // inside M-half h
          if constexpr (RPS <= 64) {
            const int i = row & (RPS - 1), jj = col & (RPS - 1);
            if ((row >> Sh::LRPS) == (col >> Sh::LRPS) && i < jj && jj < R)
              stage[(Sh::SPH * h + (row >> Sh::LRPS)) * ld_out + D + tri_offset(i, R) + (jj - i - 1)] = __float2bfloat16(z[h][4 * j + 2 * hh + c]);
          } else {
            const int i = 64 * h + row;
            if (i < col && col < R) stage[D + tri_offset(i, R) + (col - i - 1)] = __float2bfloat16(z[h][4 * j + 2 * hh + c]);
          }
        }
}

// dense pass-through (packed row 0 of each sample) + zero padding of the row tail; warp w <-> samples w, w + 4, ...
template <int D, int RPS>
__device__ __forceinline__ void fwd_stage_dense(const InterParams& p, const uint8_t* tile, __nv_bfloat16* stage, int warp, int lane) {
  using Sh = Shape<D, RPS>;
#pragma unroll
  for (int s4 = 0; s4 < (Sh::S + 3) / 4; ++s4) {
    const int s = warp + 4 * s4;
    if (Sh::S % 4 != 0 && s >= Sh::S) break;
    __nv_bfloat16* srow = stage + s * p.ld_out;
    for (int c = lane; c < Sh::CPR; c += 32) {
      const int r = s * RPS;
      reinterpret_cast<uint4*>(srow)[c] = *reinterpret_cast<const uint4*>(tile + (c >> 3) * kTileBytes + sw128_offset(r, (c & 7) * 8));
    }
    for (int c = p.out_cols + lane; c < p.ld_out; c += 32) srow[c] = __float2bfloat16(0.f);
  }
}

// Backward: D = blockdiag(S) . T, one M-half h and one N-chunk nc (NW = 64 or 128 columns, K-blocks [2 nc, 2 nc + NW / 64) of
// T). For RPS <= 64, M-half h of blockdiag(S) is zero outside K-block h, so the half is 4 x m64nNWk16 with A = S (K-major) and
// B = T consumed MN-major ([k = packed row][n = dim]; the 64-column halves of a chunk are kTileBytes apart). For RPS = 128 S is
// one dense 128 x 128 block: 8 k-steps over both K-blocks of S and all 128 rows of T.
// The halves run one after the other (64 accumulator registers instead of 128). For RPS <= 64 half h reads only rows
// [64h, 64h + 64) of K-block h of S, so the output of half 0 may already overwrite K-block 0 while half 1 runs.
template <int RPS, int NW>
__device__ __forceinline__ void bwd_mma_half(uint32_t aS, uint32_t aT, int h, int nc, float (&d)[NW / 2]) {
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < (RPS <= 64 ? 4 : 8); ++k) {
    uint64_t adesc, bdesc;
    if constexpr (RPS <= 64) {
      adesc = make_kmajor_desc(aS + h * kTileBytes + h * 8192 + k * 32);
      bdesc = make_smem_desc(aT + nc * 2 * kTileBytes + (h * 64 + k * 16) * 128, kTileBytes, 1024);
    } else {
      adesc = make_kmajor_desc(aS + (k >> 2) * kTileBytes + h * 8192 + (k & 3) * 32);
      bdesc = make_smem_desc(aT + nc * 2 * kTileBytes + k * 16 * 128, kTileBytes, 1024);
    }
    if constexpr (NW == 128) wgmma_m64n128k16<0, 1>(d, adesc, bdesc, k != 0);
    else wgmma_m64n64k16<0, 1>(d, adesc, bdesc, k != 0);
  }
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_regs(d);
}

// accumulators of half h, N-chunk nc -> global gradient rows, 4 B per store. PASS: add the pass-through gradient of
// out[:, :D] (gstage) to the dense row.
template <int D, int RPS, int NW, bool PASS>
__device__ __forceinline__ void bwd_store_direct(const InterParams& p, const float (&d)[NW / 2], const __nv_bfloat16* gstage, int b0, int h, int nc,
                                                 int R, int warp, int lane) {
  using Sh = Shape<D, RPS>;
  const int q = lane & 3;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int r = 64 * h + 16 * warp + (lane >> 2) + 8 * hh;
    const int s = r >> Sh::LRPS, i = r & (RPS - 1), b = b0 + s;
    if (b >= p.B || i >= R) continue;
#pragma unroll
    for (int j = 0; j < NW / 8; ++j) {
      if (nc * 128 + 8 * j >= D) break;
      const int col = nc * 128 + 8 * j + 2 * q;
      float v0 = d[4 * j + 2 * hh], v1 = d[4 * j + 2 * hh + 1];
      if (i == 0) {
        if (PASS) {  // dense row: add the pass-through gradient of out[:, :D]
          const __nv_bfloat162 gd = *reinterpret_cast<const __nv_bfloat162*>(gstage + s * p.ld_out + col);
          v0 += __bfloat162float(gd.x);
          v1 += __bfloat162float(gd.y);
        }
        *reinterpret_cast<__nv_bfloat162*>(reinterpret_cast<__nv_bfloat16*>(p.g_dense) + (int64_t) b * p.ld_gdense + col) = __floats2bfloat162_rn(v0, v1);
      } else if (p.gsparse_f32) {
        *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.g_sparse) + (int64_t) b * p.ld_gsparse + (i - 1) * D + col) = make_float2(v0, v1);
      } else {
        *reinterpret_cast<__nv_bfloat162*>(reinterpret_cast<__nv_bfloat16*>(p.g_sparse) + (int64_t) b * p.ld_gsparse + (i - 1) * D + col) =
            __floats2bfloat162_rn(v0, v1);
      }
    }
  }
}

// all N-chunks of half h: full 128-column chunks, then a 64-column chunk when KB is odd
template <int D, int RPS, bool PASS>
__device__ __forceinline__ void bwd_half_direct(const InterParams& p, uint32_t aS, uint32_t aT, const __nv_bfloat16* gstage, int b0, int h, int R,
                                                int warp, int lane) {
  constexpr int KB = Shape<D, RPS>::KB;
#pragma unroll 1
  for (int nc = 0; nc < KB / 2; ++nc) {
    float d[64];
    bwd_mma_half<RPS, 128>(aS, aT, h, nc, d);
    bwd_store_direct<D, RPS, 128, PASS>(p, d, gstage, b0, h, nc, R, warp, lane);
  }
  if constexpr (KB % 2 == 1) {
    float d[32];
    bwd_mma_half<RPS, 64>(aS, aT, h, KB / 2, d);
    bwd_store_direct<D, RPS, 64, PASS>(p, d, gstage, b0, h, KB / 2, R, warp, lane);
  }
}

template <int D, int RPS>
__global__ void __launch_bounds__(128, Shape<D, RPS>::kFwdCtas) interaction_fwd_kernel(const InterParams p) {
  using Sh = Shape<D, RPS>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t) 1023);
  uint8_t* tile = smem;                                            // KB x 16 KB
  __nv_bfloat16* stage = reinterpret_cast<__nv_bfloat16*>(smem + Sh::KB * kTileBytes);  // [S][ld_out] output staging
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int R = p.F + 1;

  // zero the operand tile once: padding rows (i >= R) and columns (>= D) are never written again
  for (int i = tid; i < Sh::KB * kTileBytes / 16; i += 128) reinterpret_cast<uint4*>(tile)[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  const int groups = (p.B + Sh::S - 1) / Sh::S;
  for (int g = blockIdx.x; g < groups; g += gridDim.x) {
    const int b0 = g * Sh::S;
    load_tile<D, RPS>(p, tile, b0, tid);
    fence_proxy_async();  // generic-proxy smem writes -> visible to the tensor-core (async) proxy
    __syncthreads();
    float z[2][Sh::NF / 2];
    fwd_mma_issue<D, RPS>(smem_u32(tile), z);
    mma_wait(z);
    fwd_scatter<D, RPS>(z, stage, p.ld_out, R, warp, lane);
    fwd_stage_dense<D, RPS>(p, tile, stage, warp, lane);
    __syncthreads();  // staging complete; operand tile free for the next group
    const int vec_per_row = (int) (p.ld_out >> 3);
    for (int v = tid; v < Sh::S * vec_per_row; v += 128) {
      const int s = v / vec_per_row, c = v - s * vec_per_row;
      if (b0 + s < p.B)
        reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.out) + (int64_t) (b0 + s) * p.ld_out)[c] =
            reinterpret_cast<const uint4*>(stage + s * p.ld_out)[c];
    }
    __syncthreads();
  }
}

template <int D, int RPS>
__global__ void __launch_bounds__(128, Shape<D, RPS>::kBwdCtas) interaction_bwd_kernel(const InterParams p) {
  using Sh = Shape<D, RPS>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t) 1023);
  uint8_t* tileT = smem;                          // packed X (KB K-blocks), used as MN-major B operand
  uint8_t* tileS = smem + Sh::KB * kTileBytes;    // block-diagonal S (2 K-blocks), K-major A operand
  __nv_bfloat16* gstage = reinterpret_cast<__nv_bfloat16*>(smem + (Sh::KB + 2) * kTileBytes);  // [S][ld_out] incoming gradient rows
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int R = p.F + 1;

  for (int i = tid; i < (Sh::KB + 2) * kTileBytes / 16; i += 128) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  const int groups = (p.B + Sh::S - 1) / Sh::S;
  for (int g = blockIdx.x; g < groups; g += gridDim.x) {
    const int b0 = g * Sh::S;
    load_tile<D, RPS>(p, tileT, b0, tid);
    // stage the S incoming gradient rows with coalesced 16 B loads
    {
      const int vec_per_row = (int) (p.ld_out >> 3);
      for (int v = tid; v < Sh::S * vec_per_row; v += 128) {
        const int sidx = v / vec_per_row, c = v - sidx * vec_per_row;
        uint4 val = make_uint4(0, 0, 0, 0);
        if (b0 + sidx < p.B) val = reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(p.gout) + (int64_t) (b0 + sidx) * p.ld_out)[c];
        reinterpret_cast<uint4*>(gstage + sidx * p.ld_out)[c] = val;
      }
    }
    __syncthreads();
    // S rows: thread (sample s = tid / RPS, i = tid % RPS) writes S[i][j] for all j (symmetric, zero diagonal)
    {
      const int s = tid >> Sh::LRPS, i = tid & (RPS - 1);
      const int b = b0 + s;
      const int r = s * RPS + i;
      const __nv_bfloat16* grow = gstage + s * p.ld_out + D;
      if (i < R) {
        for (int j = 0; j < R; ++j) {
          __nv_bfloat16 v = __float2bfloat16(0.f);
          if (b < p.B && j != i) {
            const int lo = min(i, j), hi = max(i, j);
            v = grow[tri_offset(lo, R) + (hi - lo - 1)];
          }
          const int k = s * RPS + j;
          *reinterpret_cast<__nv_bfloat16*>(tileS + (k >> 6) * kTileBytes + sw128_offset(r, k & 63)) = v;
        }
      }
    }
    fence_proxy_async();
    __syncthreads();
#pragma unroll 1
    for (int h = 0; h < 2; ++h) bwd_half_direct<D, RPS, true>(p, smem_u32(tileS), smem_u32(tileT), gstage, b0, h, R, warp, lane);
    __syncthreads();
  }
}


// ================================================================================================================
// Pipelined bf16 kernels (the production path): operand tiles arrive through cp.async (16 B LDGSTS, every thread has
// all of its loads in flight at once) into a DOUBLE-BUFFERED smem image, so the global->smem traffic of group g+1
// overlaps the MMA + epilogue of group g; results leave through a swizzled smem staging area with fully coalesced
// 16 B stores (the backward stores straight from registers when its output does not fit in S, D > 128 or RPS = 128).
// The kernels above (synchronous loads, per-thread 4 B stores) remain as the fp32-I/O fallback.
// ================================================================================================================

template <int D, int RPS>
__global__ void __launch_bounds__(128, Shape<D, RPS>::kFwdPipeCtas) interaction_fwd_pipe_kernel(const InterParams p) {
  using Sh = Shape<D, RPS>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t) 1023);
  uint8_t* tiles = smem;                                                                    // 2 buffers x (KB x 16 KB)
  __nv_bfloat16* stage = reinterpret_cast<__nv_bfloat16*>(smem + 2 * Sh::KB * kTileBytes);  // [S][ld_out]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int R = p.F + 1;
  for (int i = tid; i < 2 * Sh::KB * kTileBytes / 16; i += 128) reinterpret_cast<uint4*>(tiles)[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  const int groups = (p.B + Sh::S - 1) / Sh::S;
  int cur = 0;
  if ((int) blockIdx.x < groups) issue_tile_loads<D, RPS, false>(p, tiles, blockIdx.x * Sh::S, tid);
  cp_async_commit();
  for (int g = blockIdx.x; g < groups; g += gridDim.x, cur ^= 1) {
    const int b0 = g * Sh::S;
    uint8_t* tile = tiles + cur * Sh::KB * kTileBytes;
    cp_async_wait_all();
    fence_proxy_async();
    __syncthreads();  // tile[cur] landed; everyone is done with tile[cur^1] and with `stage`
    if (g + (int) gridDim.x < groups) issue_tile_loads<D, RPS, false>(p, tiles + (cur ^ 1) * Sh::KB * kTileBytes, (g + gridDim.x) * Sh::S, tid);
    cp_async_commit();
    float z[2][Sh::NF / 2];
    fwd_mma_issue<D, RPS>(smem_u32(tile), z);
    // dense passthrough + zero tail while the MMA runs
    fwd_stage_dense<D, RPS>(p, tile, stage, warp, lane);
    mma_wait(z);
    fwd_scatter<D, RPS>(z, stage, p.ld_out, R, warp, lane);
    __syncthreads();
    const int vec_per_row = (int) (p.ld_out >> 3);
#pragma unroll
    for (int s = 0; s < Sh::S; ++s) {
      if (b0 + s >= p.B) break;
      uint4* orow = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.out) + (int64_t) (b0 + s) * p.ld_out);
      const uint4* srow4 = reinterpret_cast<const uint4*>(stage + s * p.ld_out);
      for (int c = tid; c < vec_per_row; c += 128) orow[c] = srow4[c];
    }
  }
  cp_async_wait_all();
}

template <int D, int RPS, bool EXTRA>
__global__ void __launch_bounds__(128, Shape<D, RPS>::kBwdPipeCtas) interaction_bwd_pipe_kernel(const InterParams p) {
  using Sh = Shape<D, RPS>;
  constexpr int KB = Sh::KB;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t) 1023);
  uint8_t* tiles = smem;                       // T: 2 buffers x KB x 16 KB (MN-major B operand)
  uint8_t* tileS = smem + 2 * KB * kTileBytes;  // S (K-major A operand, 32 KB); re-used as the output staging area after the MMA
  __nv_bfloat16* gst = reinterpret_cast<__nv_bfloat16*>(smem + (2 * KB + 2) * kTileBytes);  // 2 x [S][ld_out]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int R = p.F + 1;
  for (int i = tid; i < 2 * KB * kTileBytes / 16; i += 128) reinterpret_cast<uint4*>(tiles)[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  const int groups = (p.B + Sh::S - 1) / Sh::S;
  const int gsz = Sh::S * (int) p.ld_out;
  int cur = 0;
  if ((int) blockIdx.x < groups) {
    issue_tile_loads<D, RPS, EXTRA>(p, tiles, blockIdx.x * Sh::S, tid);
    issue_gout_loads<Sh::S>(p, gst, blockIdx.x * Sh::S, tid);
  }
  cp_async_commit();
  // my row of the packed tile: sample s = tid / RPS, row-in-sample i = tid % RPS
  const int s = tid >> Sh::LRPS, i = tid & (RPS - 1);
  const int r = s * RPS + i;
  for (int g = blockIdx.x; g < groups; g += gridDim.x, cur ^= 1) {
    const int b0 = g * Sh::S;
    uint8_t* tileT = tiles + cur * KB * kTileBytes;
    const __nv_bfloat16* gstage = gst + cur * gsz;
    cp_async_wait_all();
    fence_proxy_async();
    __syncthreads();  // T[cur] / gout[cur] landed; copy-out of the previous group finished (staging == tileS is free)
    if (g + (int) gridDim.x < groups) {
      issue_tile_loads<D, RPS, EXTRA>(p, tiles + (cur ^ 1) * KB * kTileBytes, (g + gridDim.x) * Sh::S, tid);
      issue_gout_loads<Sh::S>(p, gst + (cur ^ 1) * gsz, (g + gridDim.x) * Sh::S, tid);
    }
    cp_async_commit();
    // ---- S row of this thread: S[i][j] = g[triangle(min,max)] (0 on the diagonal / padding); the whole 256 B row of
    //      blockdiag(S) is written (zeros outside the sample's own RPS-column block) because the staging re-use clobbers it
    {
      const __nv_bfloat16* grow = gstage + s * p.ld_out + D;
      const bool live = i < R && (b0 + s) < p.B;
      // S[i][j] = g[tri(min) + (max - min - 1)]: for j < i the offset walks down the column (stride R - j - 2), for j > i it
      // is contiguous in the row of i — no multiplications inside the loop
      uint32_t packed[RPS / 2];
      int off_lo = i - 1;
      const int off_hi = tri_offset(i, R) - (i + 1);
#pragma unroll
      for (int j2 = 0; j2 < RPS / 2; ++j2) {
        __nv_bfloat16 v[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int j = 2 * j2 + h;
          v[h] = __float2bfloat16(0.f);
          if (live && j < R && j != i) v[h] = grow[(j < i) ? off_lo : off_hi + j];
          if (EXTRA && j == R && i == 0) v[h] = __float2bfloat16(1.f);  // routes packed row R (pass-through gradient) into the dense row
          off_lo += R - j - 2;
        }
        __nv_bfloat162 hh = __halves2bfloat162(v[0], v[1]);
        packed[j2] = *reinterpret_cast<uint32_t*>(&hh);
        if constexpr (RPS == 128) {  // the row is the sample's own block: store each 16 B chunk (k in [8 cc, 8 cc + 8)) once complete
          if ((j2 & 3) == 3) {
            const int cc = j2 >> 2, c = cc & 7;
            *reinterpret_cast<uint4*>(tileS + (cc >> 3) * kTileBytes + r * 128 + (((c ^ (r & 7)) & 7) << 4)) =
                make_uint4(packed[j2 - 3], packed[j2 - 2], packed[j2 - 1], packed[j2]);
          }
        }
      }
      if constexpr (RPS <= 64) {
        // row r: K-block kb holds k in [64 kb, 64 kb + 64) as 8 chunks of 16 B; own block = k in [RPS s, RPS s + RPS)
        const int own_kb = s >> Sh::LSPH, own_c0 = (s & (Sh::SPH - 1)) * (RPS / 8);
#pragma unroll
        for (int kb = 0; kb < 2; ++kb) {
#pragma unroll
          for (int c = 0; c < 8; ++c) {
            uint4 val = make_uint4(0, 0, 0, 0);
            if (kb == own_kb && c >= own_c0 && c < own_c0 + RPS / 8) {
              const int q = (c - own_c0) * 4;
              val = make_uint4(packed[q], packed[q + 1], packed[q + 2], packed[q + 3]);
            }
            *reinterpret_cast<uint4*>(tileS + kb * kTileBytes + r * 128 + (((c ^ (r & 7)) & 7) << 4)) = val;
          }
        }
      }
    }
    fence_proxy_async();
    __syncthreads();
    if constexpr (!Sh::kStageInS) {
#pragma unroll 1
      for (int h = 0; h < 2; ++h) bwd_half_direct<D, RPS, !EXTRA>(p, smem_u32(tileS), smem_u32(tileT), gstage, b0, h, R, warp, lane);
    } else {
      // ---- per half: MMA, then registers -> bf16 -> swizzled staging ([128 rows][8 KB chunks of 16 B], chunk ^= row). The
      //      staging rows of half h are K-block h of S, which only half h reads: its wgmma has retired when the stores start.
      constexpr int NW = 64 * KB, CMASK = 8 * KB - 1;
      uint8_t* ostage = tileS;
      const int q = lane & 3;
#pragma unroll 1
      for (int h = 0; h < 2; ++h) {
        float d[NW / 2];
        bwd_mma_half<RPS, NW>(smem_u32(tileS), smem_u32(tileT), h, 0, d);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int rr = 64 * h + 16 * warp + (lane >> 2) + 8 * hh;
#pragma unroll
          for (int j = 0; j < NW / 8; ++j) {
            float v0 = d[4 * j + 2 * hh], v1 = d[4 * j + 2 * hh + 1];
            if (!EXTRA && (rr & (RPS - 1)) == 0) {  // R == RPS: no spare packed row, add the pass-through gradient of out[:, :D] here
              const __nv_bfloat162 gd = *reinterpret_cast<const __nv_bfloat162*>(gstage + (rr >> Sh::LRPS) * p.ld_out + 8 * j + 2 * q);
              v0 += __bfloat162float(gd.x);
              v1 += __bfloat162float(gd.y);
            }
            *reinterpret_cast<__nv_bfloat162*>(ostage + rr * (KB * 128) + (((j ^ rr) & CMASK) << 4) + 4 * q) = __floats2bfloat162_rn(v0, v1);
          }
        }
      }
      __syncthreads();
      // ---- coalesced copy-out: CPR consecutive threads write one D-column gradient row
      if constexpr (Sh::kFixedChunk) {
        constexpr int RSTEP = Sh::RSTEP;
        const int ch = tid & (Sh::CPR - 1), i0 = tid >> Sh::LCPR;
        __nv_bfloat16* gd_base = reinterpret_cast<__nv_bfloat16*>(p.g_dense) + ch * 8;
        __nv_bfloat16* gs_base = reinterpret_cast<__nv_bfloat16*>(p.g_sparse) + ch * 8 - D;
#pragma unroll
        for (int s4 = 0; s4 < Sh::S; ++s4) {
          const int b = b0 + s4;
          if (b >= p.B) break;
#pragma unroll
          for (int k = 0; k < RPS / RSTEP; ++k) {
            const int ii = i0 + RSTEP * k;
            if (ii >= R) break;
            const uint4 val = *reinterpret_cast<const uint4*>(ostage + (s4 * RPS + ii) * (KB * 128) + (((ch ^ ii) & CMASK) << 4));
            __nv_bfloat16* dst = (ii == 0) ? gd_base + (int64_t) b * p.ld_gdense : gs_base + (int64_t) b * p.ld_gsparse + (int64_t) ii * D;
            *reinterpret_cast<uint4*>(dst) = val;
          }
        }
      } else {
#pragma unroll
        for (int k = 0; k < Sh::CPR; ++k) {
          const int c = tid + 128 * k;
          const int rr = (int) ((unsigned) c / Sh::CPR), ch = (int) ((unsigned) c % Sh::CPR);
          const int ii = rr & (RPS - 1), b = b0 + (rr >> Sh::LRPS);
          if (ii >= R || b >= p.B) continue;
          const uint4 val = *reinterpret_cast<const uint4*>(ostage + rr * (KB * 128) + (((ch ^ rr) & CMASK) << 4));
          __nv_bfloat16* dst = (ii == 0) ? reinterpret_cast<__nv_bfloat16*>(p.g_dense) + (int64_t) b * p.ld_gdense
                                         : reinterpret_cast<__nv_bfloat16*>(p.g_sparse) + (int64_t) b * p.ld_gsparse + (int64_t) (ii - 1) * D;
          *reinterpret_cast<uint4*>(dst + ch * 8) = val;
        }
      }
    }
  }
  cp_async_wait_all();
}

// ---- host side ---------------------------------------------------------------------------------------------------------
struct DeviceLimits {
  int sms, smem_optin, smem_per_sm, smem_reserved;
};

inline const DeviceLimits& device_limits() {
  static DeviceLimits l = [] {
    DeviceLimits d = {};
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&d.sms, cudaDevAttrMultiProcessorCount, dev);
    cudaDeviceGetAttribute(&d.smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    cudaDeviceGetAttribute(&d.smem_per_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev);
    cudaDeviceGetAttribute(&d.smem_reserved, cudaDevAttrReservedSharedMemoryPerBlock, dev);
    return d;
  }();
  return l;
}

// Launch a persistent kernel: `max_ctas` CTAs per SM (its __launch_bounds__), fewer when `smem` bytes of dynamic shared memory
// per CTA do not fit that many. Returns -22 without launching when one CTA needs more than the device's opt-in limit.
inline int launch_persistent(void (*kernel)(const InterParams), bool& configured, int max_ctas, int smem, int groups, const InterParams& p,
                             cudaStream_t stream) {
  const DeviceLimits& lim = device_limits();
  if (smem > lim.smem_optin) return -22;
  if (!configured) {
    TRB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, lim.smem_optin));
    configured = true;
  }
  int ctas = lim.smem_per_sm / (smem + lim.smem_reserved);
  ctas = ctas < 1 ? 1 : (ctas < max_ctas ? ctas : max_ctas);
  const int grid = groups < ctas * lim.sms ? groups : ctas * lim.sms;
  kernel<<<grid, 128, smem, stream>>>(p);
  TRB_CHECK_LAUNCH();
  return 0;
}

template <int D, int RPS>
int launch_fwd(const InterParams& p, cudaStream_t stream) {
  using Sh = Shape<D, RPS>;
  const int groups = (p.B + Sh::S - 1) / Sh::S;
  if (!p.sparse_f32 && p.ld_dense % 8 == 0 && p.ld_sparse % 8 == 0) {
    static bool cfg_p = false;
    const int smem_p = 2 * Sh::KB * kTileBytes + Sh::S * (int) p.ld_out * 2 + 64 + 1024;
    return launch_persistent(interaction_fwd_pipe_kernel<D, RPS>, cfg_p, Sh::kFwdPipeCtas, smem_p, groups, p, stream);
  }
  static bool cfg = false;
  const int smem = Sh::KB * kTileBytes + Sh::S * (int) p.ld_out * 2 + 64 + 1024;
  return launch_persistent(interaction_fwd_kernel<D, RPS>, cfg, Sh::kFwdCtas, smem, groups, p, stream);
}

template <int D, int RPS>
int launch_bwd(const InterParams& p, cudaStream_t stream) {
  using Sh = Shape<D, RPS>;
  const int groups = (p.B + Sh::S - 1) / Sh::S;
  if (!p.sparse_f32 && !p.gsparse_f32 && p.ld_dense % 8 == 0 && p.ld_sparse % 8 == 0 && p.ld_gdense % 8 == 0 && p.ld_gsparse % 8 == 0 &&
      p.ld_out % 8 == 0) {
    static bool cfg_x = false, cfg_p = false;
    const int smem_p = (2 * Sh::KB + 2) * kTileBytes + 2 * Sh::S * (int) p.ld_out * 2 + 64 + 1024;
    if (p.F + 1 < RPS) return launch_persistent(interaction_bwd_pipe_kernel<D, RPS, true>, cfg_x, Sh::kBwdPipeCtas, smem_p, groups, p, stream);
    return launch_persistent(interaction_bwd_pipe_kernel<D, RPS, false>, cfg_p, Sh::kBwdPipeCtas, smem_p, groups, p, stream);
  }
  static bool cfg = false;
  const int smem = (Sh::KB + 2) * kTileBytes + Sh::S * (int) p.ld_out * 2 + 64 + 1024;
  return launch_persistent(interaction_bwd_kernel<D, RPS>, cfg, Sh::kBwdCtas, smem, groups, p, stream);
}

// the packing of R = F + 1 rows: the smallest RPS in {16, 32, 64, 128} with R <= RPS
template <int D>
int launch_fwd_d(const InterParams& p, cudaStream_t stream) {
  const int R = p.F + 1;
  if (R <= 16) return launch_fwd<D, 16>(p, stream);
  if (R <= 32) return launch_fwd<D, 32>(p, stream);
  if (R <= 64) return launch_fwd<D, 64>(p, stream);
  return launch_fwd<D, 128>(p, stream);
}

template <int D>
int launch_bwd_d(const InterParams& p, cudaStream_t stream) {
  const int R = p.F + 1;
  if (R <= 16) return launch_bwd<D, 16>(p, stream);
  if (R <= 32) return launch_bwd<D, 32>(p, stream);
  if (R <= 64) return launch_bwd<D, 64>(p, stream);
  return launch_bwd<D, 128>(p, stream);
}

}  // namespace

// one group of four widths: D0, D0 + 16, D0 + 32, D0 + 48
#define TRB_INTERACTION_GROUP(NAME, D0)                                                    \
  namespace trb {                                                                          \
  int interaction_fwd_##NAME(const InterParams& p, int D, cudaStream_t stream) {           \
    switch (D) {                                                                           \
      case D0: return launch_fwd_d<D0>(p, stream);                                         \
      case D0 + 16: return launch_fwd_d<D0 + 16>(p, stream);                               \
      case D0 + 32: return launch_fwd_d<D0 + 32>(p, stream);                               \
      case D0 + 48: return launch_fwd_d<D0 + 48>(p, stream);                               \
      default: return -20;                                                                 \
    }                                                                                      \
  }                                                                                        \
  int interaction_bwd_##NAME(const InterParams& p, int D, cudaStream_t stream) {           \
    switch (D) {                                                                           \
      case D0: return launch_bwd_d<D0>(p, stream);                                         \
      case D0 + 16: return launch_bwd_d<D0 + 16>(p, stream);                               \
      case D0 + 32: return launch_bwd_d<D0 + 32>(p, stream);                               \
      case D0 + 48: return launch_bwd_d<D0 + 48>(p, stream);                               \
      default: return -20;                                                                 \
    }                                                                                      \
  }                                                                                        \
  }
