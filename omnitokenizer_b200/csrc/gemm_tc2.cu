// GEMM v2: 3xTF32 error-compensated GEMM on sm_90a wgmma (the kernel lives in gemm_wgmma.cuh, shared with gemm_f16.cu).
//
//   C[M,N] = A[M,K] . W[N,K]^T (+bias)(+residual) | GEGLU | rope+l2norm+scale,   fp32 in / out, fp32-grade accuracy.
//
// A arrives as fp32 by TMA and each consumer warpgroup splits its 64 rows into tf32 hi / lo in shared memory; W arrives
// pre-split (hi = tf32(W), lo = W - hi).  Three tf32 MMAs per k-step (A_lo.W_hi + A_hi.W_lo + A_hi.W_hi) accumulate into
// one fp32 accumulator in registers.
#include "gemm_wgmma.cuh"

namespace omt {

int launch_gemm_tc2(const GemmArgs& g, const float* W_lo, int epilogue, cudaStream_t st, const float* A2, int n_split) {
  using namespace wgg;
  OMT_REQUIRE(g.K % 32 == 0 && g.lda % 4 == 0, "omt_linear(wgmma 3xTF32): K=%d must be a multiple of 32", g.K);
  if (g.a_seg > 0) {
    OMT_REQUIRE(g.a_seg % 64 == 0 && g.M % g.a_seg == 0, "omt_linear(wgmma 3xTF32): A row-map segment %d must be a multiple of 64 dividing M=%d", g.a_seg, g.M);
  }
  if (A2 != nullptr) OMT_REQUIRE(n_split > 0 && n_split % 128 == 0, "omt_linear2: n_split=%d must be a multiple of 128", n_split);
  const int n_pad = (g.N + 127) / 128 * 128;
  const CUtensorMapDataType f32 = CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  CUtensorMap maps[6];
  int rc;
  if ((rc = row_map(&maps[0], f32, 4, g.A, g.lda, g.M, g.K, g.a_seg, g.a_seg_stride, g.a_seg_off))) return rc;
  if ((rc = row_map(&maps[2], f32, 4, A2 != nullptr ? A2 : g.A, g.lda, g.M, g.K, g.a_seg, g.a_seg_stride, g.a_seg_off))) return rc;
  maps[1] = maps[0]; maps[3] = maps[2];       // no lo planes: A is split in shared memory
  if ((rc = w_map(&maps[4], f32, 4, g.W, n_pad, g.K))) return rc;
  if ((rc = w_map(&maps[5], f32, 4, W_lo, n_pad, g.K))) return rc;
  Args a{};
  a.M = g.M; a.N = g.N; a.K = g.K;
  a.num_m_blk = (g.M + BM - 1) / BM;
  a.n_split = A2 != nullptr ? n_split : 0x7fffffff;
  a.a_seg = g.a_seg; a.a_seg_stride = g.a_seg_stride; a.a_seg_off = g.a_seg_off;
  a.c = g.C; a.ldc = g.ldc;
  a.c_seg = g.c_seg; a.c_seg_stride = g.c_seg_stride; a.c_seg_off = g.c_seg_off;
  a.bias = g.bias; a.residual = g.residual; a.ldr = g.ldr;
  a.rope_cos = g.rope_cos; a.rope_sin = g.rope_sin; a.q_scale = g.q_scale; a.k_scale = g.k_scale;
  a.qk_cols = g.qk_cols; a.tokens = g.tokens > 0 ? g.tokens : 1;
  if (epilogue == OMT_EPI_QKV) return launch<true, 1, OMT_EPI_QKV>(maps, a, st);
  if (epilogue == OMT_EPI_GEGLU) return launch<true, 1, OMT_EPI_GEGLU>(maps, a, st);
  return launch<true, 1, OMT_EPI_NONE>(maps, a, st);
}

}  // namespace omt
