// DLRM dot-interaction forward / backward on wgmma tensor cores (sm_90a): C ABI and the D = 80 ... 128 instances.
//
//   X_b = [dense_b ; sparse_b]            (R = F+1 rows, D columns)
//   out_b = [dense_b , strict-upper-triangle(X_b X_b^T)]         (reference models/dlrm.py:210-222)
//
// Shapes: D % 16 == 0 with 16 <= D <= 256, and 1 <= F <= 127 (R <= 128 rows fit one 128-row operand tile). The kernels
// (interaction.cuh) are templates over D and the packing RPS: samples with R <= 16 / 32 / 64 / 128 get 16 / 32 / 64 / 128 rows
// of the tile, so 8 / 4 / 2 / 1 of them share one MMA tile. Other shapes return -20; the caller runs the interaction in
// PyTorch (ops/dense.py: dot_interaction).
#include "interaction.cuh"

TRB_INTERACTION_GROUP(d80_128, 80)

namespace {

bool shape_ok(int F, int D) { return D % 16 == 0 && D >= 16 && D <= 256 && F >= 1 && F <= 127; }

int dispatch_fwd(const InterParams& p, int D, cudaStream_t stream) {
  if (D <= 64) return interaction_fwd_d16_64(p, D, stream);
  if (D <= 128) return interaction_fwd_d80_128(p, D, stream);
  if (D <= 192) return interaction_fwd_d144_192(p, D, stream);
  return interaction_fwd_d208_256(p, D, stream);
}

int dispatch_bwd(const InterParams& p, int D, cudaStream_t stream) {
  if (D <= 64) return interaction_bwd_d16_64(p, D, stream);
  if (D <= 128) return interaction_bwd_d80_128(p, D, stream);
  if (D <= 192) return interaction_bwd_d144_192(p, D, stream);
  return interaction_bwd_d208_256(p, D, stream);
}

}  // namespace

// out[b] = [dense_b, triu(X_b X_b^T, 1)] with ld_out >= D + R(R-1)/2 (multiple of 8, tail zero filled).
// Returns -20 for a shape the kernels do not cover, -21 for a bad ld_out, -22 when the shared memory of one CTA would exceed the
// device's opt-in limit.
TRB_API int trb_interaction_fwd(const void* dense, int64_t ld_dense, const void* sparse, int64_t ld_sparse, int sparse_f32, void* out,
                                int64_t ld_out, int B, int F, int D, cudaStream_t stream) {
  if (!shape_ok(F, D)) return -20;
  if (B == 0) return 0;
  InterParams p = {};
  p.dense = dense; p.ld_dense = ld_dense; p.sparse = sparse; p.ld_sparse = ld_sparse; p.sparse_f32 = sparse_f32;
  p.out = out; p.ld_out = ld_out; p.B = B; p.F = F; p.out_cols = D + (F + 1) * F / 2;
  if (ld_out % 8 || ld_out < p.out_cols) return -21;
  return dispatch_fwd(p, D, stream);
}

TRB_API int trb_interaction_bwd(const void* dense, int64_t ld_dense, const void* sparse, int64_t ld_sparse, int sparse_f32, const void* gout,
                                int64_t ld_out, void* g_dense, int64_t ld_gdense, void* g_sparse, int64_t ld_gsparse, int gsparse_f32, int B,
                                int F, int D, cudaStream_t stream) {
  if (!shape_ok(F, D)) return -20;
  if (B == 0) return 0;
  InterParams p = {};
  p.dense = dense; p.ld_dense = ld_dense; p.sparse = sparse; p.ld_sparse = ld_sparse; p.sparse_f32 = sparse_f32;
  p.gout = gout; p.ld_out = ld_out; p.B = B; p.F = F; p.out_cols = D + (F + 1) * F / 2;
  p.g_dense = g_dense; p.ld_gdense = ld_gdense; p.g_sparse = g_sparse; p.ld_gsparse = ld_gsparse; p.gsparse_f32 = gsparse_f32;
  return dispatch_bwd(p, D, stream);
}
