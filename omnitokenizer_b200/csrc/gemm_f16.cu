// GEMM v3 ("f16x3"): wgmma f16 GEMM on pre-split 16-bit operands (the kernel lives in gemm_wgmma.cuh).
//
//   C[M,N] = A[M,K] . W[N,K]^T (+bias)(+residual) | GEGLU | rope+l2norm+scale,   fp32-grade accuracy.
//
// Every fp32 operand x is carried as TWO fp16 planes, hi = fp16(x) and lo = fp16((x - hi) * 2^11) (omt_common.cuh:
// 11 + 11 significant bits, error <= 2^-23 |x|), written ONCE by whatever kernel produced x (LayerNorm, the attention
// cores, the GEGLU epilogue of this kernel; weights at pack time).  The product is
//       A.W ~= A_hi.W_hi + 2^-11 (A_hi.W_lo + A_lo.W_hi)
// three f16 wgmmas per k-step: the first into the MAIN fp32 accumulator, the two cross products into a second one that
// the epilogue folds in with an exact power-of-two scale.  Against the 3xTF32 kernel (gemm_tc2.cu):
//   * 16-bit MMAs run at twice the tf32 rate -> the exactness tax drops from 3 to 1.5 tf32-equivalents per product;
//   * the operands arrive in their final shared-memory form by TMA: no split in shared memory;
//   * W_hi / W_lo are half the bytes, A_hi + A_lo the same bytes as the fp32 activation.
//
// NACC = 1, the ROW-SCALED form (omt_common.cuh): when the A planes come from a producer that saw whole rows (LayerNorm,
// patch gather) they carry a per-row power-of-two scale and an UNSCALED lo plane, the weights a per-matrix one; all three
// products then share ONE accumulator.  The epilogue multiplies by the exact inverse scales (a_rs[row] * w_scale).
//
// omt_linear_h1 ("f16x1", the throughput mode): the same argument block without the lo planes.  Every k-step is ONE f16
// wgmma A_hi.W_hi into the fp32 accumulator (11 significant bits per operand, like single-pass TF32); row-scaled and
// uniform-scaled A take the same epilogue factor as above, the 2^11 form (unscaled hi planes) none.  Output planes are
// written hi only.
#include "gemm_wgmma.cuh"

namespace omt {

int g_f16_bn = 0;   // omt_set_option("f16_bn", 0|128|256): accepted for compatibility; the wgmma kernel always uses 128-wide tiles

// A planes: [M, lda] fp16; W planes: [n_pad, K] fp16 (rows padded to 256); C fp32 (plain / QKV) or U planes (GEGLU / QKV planes)
// `who` names the entry point in error messages; h1: the single-product kernel (no lo planes)
static int launch_gemm_f16(const omt_linear_h_args& a, cudaStream_t st, const char* who, bool h1) {
  using namespace wgg;
  const bool rs = a.a_rs != nullptr || a.a_rs_uniform > 0.f;   // row-scaled planes: one accumulator
  OMT_REQUIRE(a.K % 64 == 0 && a.lda % 8 == 0, "%s: K=%d must be a multiple of 64 and lda %% 8 == 0", who, a.K);
  if (a.a_seg > 0)
    OMT_REQUIRE(a.a_seg % 64 == 0 && a.M % a.a_seg == 0, "%s: A row-map segment %d must be a multiple of 64 dividing M=%d", who, a.a_seg, a.M);
  if (a.c_seg > 0)
    OMT_REQUIRE(a.c_seg % 32 == 0 && a.M % a.c_seg == 0, "%s: C row-map segment %d must be a multiple of 32 dividing M=%d", who, a.c_seg, a.M);
  OMT_REQUIRE(a.N % 32 == 0, "%s: N=%d must be a multiple of 32", who, a.N);
  if (a.a2_hi != nullptr) OMT_REQUIRE(a.n_split > 0 && a.n_split % 128 == 0, "%s: n_split=%d must be a multiple of 128", who, a.n_split);
  const int n_pad = (a.N + 255) / 256 * 256;
  const CUtensorMapDataType f16 = CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const bool dual = a.a2_hi != nullptr;
  CUtensorMap maps[8];
  int rc;
  if (a.epilogue == OMT_EPI_GEGLU || a.epilogue == OMT_EPI_QKV_PLANES) {   // output planes, written by TMA stores
    const bool geglu = a.epilogue == OMT_EPI_GEGLU;
    const int cols = geglu ? a.N / 2 : a.N;
    const int seg = geglu ? a.c_seg : 0;
    if ((rc = row_map(&maps[6], f16, 2, a.u_hi, a.ldu, a.M, cols, seg, a.c_seg_stride, a.c_seg_off, 32))) return rc;
    if (h1) maps[7] = maps[6];
    else if ((rc = row_map(&maps[7], f16, 2, a.u_lo, a.ldu, a.M, cols, seg, a.c_seg_stride, a.c_seg_off, 32))) return rc;
  }
  if ((rc = row_map(&maps[0], f16, 2, a.a_hi, a.lda, a.M, a.K, a.a_seg, a.a_seg_stride, a.a_seg_off))) return rc;
  if ((rc = row_map(&maps[2], f16, 2, dual ? a.a2_hi : a.a_hi, a.lda, a.M, a.K, a.a_seg, a.a_seg_stride, a.a_seg_off))) return rc;
  if ((rc = w_map(&maps[4], f16, 2, a.w_hi, n_pad, a.K))) return rc;
  if (h1) {          // the lo maps are never loaded
    maps[1] = maps[0]; maps[3] = maps[2]; maps[5] = maps[4];
  } else {
    if ((rc = row_map(&maps[1], f16, 2, a.a_lo, a.lda, a.M, a.K, a.a_seg, a.a_seg_stride, a.a_seg_off))) return rc;
    if ((rc = row_map(&maps[3], f16, 2, dual ? a.a2_lo : a.a_lo, a.lda, a.M, a.K, a.a_seg, a.a_seg_stride, a.a_seg_off))) return rc;
    if ((rc = w_map(&maps[5], f16, 2, a.w_lo, n_pad, a.K))) return rc;
  }
  Args g{};
  g.M = a.M; g.N = a.N; g.K = a.K;
  g.num_m_blk = (a.M + BM - 1) / BM;
  g.n_split = dual ? a.n_split : 0x7fffffff;
  g.a_seg = a.a_seg; g.a_seg_stride = a.a_seg_stride; g.a_seg_off = a.a_seg_off;
  g.a_rs = a.a_rs; g.a2_rs = dual ? a.a2_rs : a.a_rs; g.w_scale = a.w_scale;
  g.a_rs_uniform = a.a_rs_uniform; g.u_scale = a.u_scale;
  g.c = a.c; g.ldc = a.ldc;
  g.c_seg = a.c_seg; g.c_seg_stride = a.c_seg_stride; g.c_seg_off = a.c_seg_off;
  g.bias = a.bias; g.residual = a.residual; g.ldr = a.ldr;
  g.u_hi = a.u_hi; g.u_lo = a.u_lo; g.ldu = a.ldu;
  g.rope_cos = a.rope_cos; g.rope_sin = a.rope_sin; g.q_scale = a.q_scale; g.k_scale = a.k_scale;
  g.qk_cols = a.qk_cols; g.tokens = a.tokens > 0 ? a.tokens : 1;
  g.q_ps = a.q_plane_scale; g.k_ps = a.k_plane_scale; g.vinv = a.vinv;
  if (h1 && !rs) { g.a_rs_uniform = 1.f; g.w_scale = 1.f; }   // 2^11 form: unscaled hi planes, exact factor 1
#define OMT_F16_LAUNCH(EPI_) (h1 ? launch<false, 1, EPI_, true>(maps, g, st) \
                              : rs ? launch<false, 1, EPI_>(maps, g, st) : launch<false, 2, EPI_>(maps, g, st))
  if (a.epilogue == OMT_EPI_QKV) return OMT_F16_LAUNCH(OMT_EPI_QKV);
  if (a.epilogue == OMT_EPI_QKV_PLANES) return OMT_F16_LAUNCH(OMT_EPI_QKV_PLANES);
  if (a.epilogue == OMT_EPI_GEGLU) return OMT_F16_LAUNCH(OMT_EPI_GEGLU);
  return OMT_F16_LAUNCH(OMT_EPI_NONE);
#undef OMT_F16_LAUNCH
}

}  // namespace omt

using namespace omt;

// Checks shared by omt_linear_h and omt_linear_h1 (h1: every lo plane must be NULL, the hi planes alone are required).
static int check_linear_h(const omt_linear_h_args* a, const char* who, bool h1) {
  OMT_REQUIRE(a != nullptr, "%s: null argument block", who);
  if (h1) {
    OMT_REQUIRE(a->a_hi && a->w_hi, "%s: null operand plane", who);
    OMT_REQUIRE(!a->a_lo && !a->a2_lo && !a->w_lo && !a->u_lo,
                "%s: lo planes must be NULL (the single-product GEMM reads and writes hi planes only)", who);
  } else {
    OMT_REQUIRE(a->a_hi && a->a_lo && a->w_hi && a->w_lo, "%s: null operand plane", who);
    OMT_REQUIRE((a->a2_hi == nullptr) == (a->a2_lo == nullptr), "%s: the second A needs both planes", who);
  }
  OMT_REQUIRE(a->a2_hi == nullptr || ((a->a_rs == nullptr) == (a->a2_rs == nullptr)), "%s: both A operands must use the same plane format", who);
  OMT_REQUIRE((a->a_rs == nullptr && !(a->a_rs_uniform > 0.f)) || (a->w_scale > 0.f && a->w_scale < 3.0e38f), "%s: row-scaled planes need the weight scale", who);
  OMT_REQUIRE(a->a_rs == nullptr || !(a->a_rs_uniform > 0.f), "%s: per-row and uniform A scales are exclusive", who);
  OMT_REQUIRE(!(a->a_rs_uniform > 0.f) || a->a2_hi == nullptr, "%s: the uniform A scale has no dual-A form", who);
  OMT_REQUIRE(a->M >= 0 && a->N > 0 && a->K > 0, "%s: bad shape M=%d N=%d K=%d", who, a->M, a->N, a->K);
  OMT_REQUIRE(a->epilogue == OMT_EPI_NONE || a->epilogue == OMT_EPI_GEGLU || a->epilogue == OMT_EPI_QKV || a->epilogue == OMT_EPI_QKV_PLANES,
              "%s: unknown epilogue %d", who, a->epilogue);
  const bool u_lo_ok = h1 || a->u_lo;
  if (a->epilogue == OMT_EPI_QKV_PLANES) {
    OMT_REQUIRE(a->u_hi && u_lo_ok && a->vinv && a->ldu % 8 == 0 && a->q_plane_scale > 0.f && a->k_plane_scale > 0.f,
                "%s: the QKV-planes epilogue writes u_hi / u_lo [M, N] (ldu %% 8 == 0), vinv and needs the q / k plane scales", who);
    OMT_REQUIRE(((uintptr_t)a->u_hi | (uintptr_t)a->u_lo) % 16 == 0, "%s: output planes must be 16-byte aligned", who);
  } else if (a->epilogue == OMT_EPI_GEGLU) {
    OMT_REQUIRE(a->u_hi && u_lo_ok && a->ldu % 8 == 0 && a->residual == nullptr && a->bias == nullptr,
                "%s: GEGLU writes the U planes (ldu %% 8 == 0) and takes no bias / residual", who);
    OMT_REQUIRE(((uintptr_t)a->u_hi | (uintptr_t)a->u_lo) % 16 == 0, "%s: U planes must be 16-byte aligned", who);
  } else {
    OMT_REQUIRE(a->c != nullptr && a->ldc % 4 == 0 && (uintptr_t)a->c % 16 == 0, "%s: C must be 16-byte aligned with ldc %% 4 == 0", who);
    OMT_REQUIRE(a->residual == nullptr || (a->ldr % 4 == 0 && (uintptr_t)a->residual % 16 == 0), "%s: bad residual", who);
    OMT_REQUIRE(a->bias == nullptr || (uintptr_t)a->bias % 16 == 0, "%s: bias must be 16-byte aligned", who);
  }
  if (a->epilogue == OMT_EPI_QKV || a->epilogue == OMT_EPI_QKV_PLANES) {
    OMT_REQUIRE(a->q_scale && a->k_scale && a->qk_cols > 0 && a->qk_cols % 128 == 0 && a->qk_cols <= a->N && a->tokens > 0 &&
                a->tokens % 32 == 0, "%s: bad q/k preparation arguments", who);
    OMT_REQUIRE((a->rope_cos == nullptr) == (a->rope_sin == nullptr), "%s: cos/sin must both be given", who);
    OMT_REQUIRE(a->bias == nullptr && a->residual == nullptr && a->N % 64 == 0, "%s: the QKV epilogue takes no bias / residual", who);
  }
  OMT_REQUIRE(((uintptr_t)a->a_hi | (uintptr_t)a->a_lo | (uintptr_t)a->a2_hi | (uintptr_t)a->a2_lo | (uintptr_t)a->w_hi | (uintptr_t)a->w_lo) % 16 == 0,
              "%s: operand planes must be 16-byte aligned", who);
  return OMT_OK;
}

extern "C" int omt_linear_h(const omt_linear_h_args* a, omt_stream_t stream) {
  OMT_ENTER();
  int rc = check_linear_h(a, "omt_linear_h", false);
  if (rc != OMT_OK) return rc;
  if (a->M == 0) return OMT_OK;
  return launch_gemm_f16(*a, (cudaStream_t)stream, "omt_linear_h", false);
}

extern "C" int omt_linear_h1(const omt_linear_h_args* a, omt_stream_t stream) {
  OMT_ENTER();
  int rc = check_linear_h(a, "omt_linear_h1", true);
  if (rc != OMT_OK) return rc;
  if (a->M == 0) return OMT_OK;
  return launch_gemm_f16(*a, (cudaStream_t)stream, "omt_linear_h1", true);
}
