// Exact-fp32 CUDA-core GEMM (the parity anchor for every nn.Linear on the path):
//   C[M,N] = A[M,K] . W[N,K]^T (+bias) (+residual) | GEGLU-paired epilogue.
// 128x128x8 tiles, 256 threads, 8x8 register blocking, register-staged double buffering.
// Both operands are K-major in HBM; tiles are transposed on the way into shared memory so the
// inner product reads conflict-free float4 fragments.
#include "omt_common.cuh"

namespace omt {

constexpr int BM = 128, BN = 128, BK = 8;
constexpr int LDS_ = 132;   // padded row stride of the transposed tiles (floats)


template <int EPI>
__global__ void __launch_bounds__(256, 2) gemm_fp32_kernel(const GemmArgs g) {
  pdl_sync();
  __shared__ __align__(16) float As[2][BK * LDS_];
  __shared__ __align__(16) float Ws[2][BK * LDS_];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;

  // global -> register staging: one float4 of A and one of W per thread per k-tile
  const int lrow = tid >> 1, lkq = (tid & 1) * 4;
  int am = m0 + lrow;
  if (am >= g.M) am = g.M - 1;
  const float* abase = (g.A2 != nullptr && n0 >= g.n_split) ? g.A2 : g.A;
  const float* aptr = abase + map_row(am, g.a_seg, g.a_seg_stride, g.a_seg_off) * g.lda + lkq;
  const float* wptr = g.W + (size_t)(n0 + lrow) * g.K + lkq;   // W rows are padded to a BN multiple

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  float4 ra = *reinterpret_cast<const float4*>(aptr);
  float4 rw = *reinterpret_cast<const float4*>(wptr);
  auto stage = [&](int buf) {
    float* as = As[buf] + lkq * LDS_ + lrow;
    as[0] = ra.x; as[LDS_] = ra.y; as[2 * LDS_] = ra.z; as[3 * LDS_] = ra.w;
    float* ws = Ws[buf] + lkq * LDS_ + lrow;
    ws[0] = rw.x; ws[LDS_] = rw.y; ws[2 * LDS_] = rw.z; ws[3 * LDS_] = rw.w;
  };
  stage(0);
  __syncthreads();

  const int KT = g.K / BK;
  for (int kt = 0; kt < KT; ++kt) {
    const int cur = kt & 1;
    if (kt + 1 < KT) {
      ra = *reinterpret_cast<const float4*>(aptr + (kt + 1) * BK);
      rw = *reinterpret_cast<const float4*>(wptr + (kt + 1) * BK);
    }
    const float* as = As[cur] + ty * 4;
    const float* ws = Ws[cur] + tx * 4;
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(as + k * LDS_);
      const float4 a1 = *reinterpret_cast<const float4*>(as + k * LDS_ + 64);
      const float4 b0 = *reinterpret_cast<const float4*>(ws + k * LDS_);
      const float4 b1 = *reinterpret_cast<const float4*>(ws + k * LDS_ + 64);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < KT) {
      stage(cur ^ 1);
      __syncthreads();
    }
  }

  // epilogue
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + (i >> 2) * 64 + ty * 4 + (i & 3);
    if (m >= g.M) continue;
    const long long prow = map_row(m, g.c_seg, g.c_seg_stride, g.c_seg_off);
#pragma unroll
    for (int jg = 0; jg < 2; ++jg) {
      const int n = n0 + jg * 64 + tx * 4;
      if (n >= g.N) continue;
      float4 v = make_float4(acc[i][jg * 4 + 0], acc[i][jg * 4 + 1], acc[i][jg * 4 + 2], acc[i][jg * 4 + 3]);
      if (g.bias != nullptr) {
        const float4 bb = *reinterpret_cast<const float4*>(g.bias + n);
        v.x += bb.x; v.y += bb.y; v.z += bb.z; v.w += bb.w;
      }
      if (EPI == OMT_EPI_GEGLU) {
        float2 o;
        o.x = gelu_erf(v.y) * v.x;
        o.y = gelu_erf(v.w) * v.z;
        *reinterpret_cast<float2*>(g.C + prow * g.ldc + (n >> 1)) = o;
      } else {
        if (g.residual != nullptr) {
          const float4 rr = *reinterpret_cast<const float4*>(g.residual + prow * g.ldr + n);
          v.x += rr.x; v.y += rr.y; v.z += rr.z; v.w += rr.w;
        }
        *reinterpret_cast<float4*>(g.C + prow * g.ldc + n) = v;
      }
    }
  }
}

int launch_gemm_fp32(const GemmArgs& g, int epilogue, cudaStream_t st) {
  dim3 grid((g.N + BN - 1) / BN, (g.M + BM - 1) / BM), block(256);
  if (epilogue == OMT_EPI_GEGLU)
    gemm_fp32_kernel<OMT_EPI_GEGLU><<<grid, block, 0, st>>>(g);
  else
    gemm_fp32_kernel<OMT_EPI_NONE><<<grid, block, 0, st>>>(g);
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

int launch_gemm_tc2(const GemmArgs& g, const float* W_lo, int epilogue, cudaStream_t st, const float* A2, int n_split);

}  // namespace omt

using namespace omt;

struct QkPrep { const float* q_scale; const float* k_scale; const float* cos; const float* sin; int qk_cols; int tokens; };

static int linear_impl(const QkPrep* qk, const float* A, const float* A2, int n_split, int lda, int a_seg, int a_seg_stride, int a_seg_off,
                          const float* W, const float* W_lo, float* C, int ldc, int c_seg, int c_seg_stride,
                          int c_seg_off, int M, int N, int K, const float* bias, const float* residual,
                          int ldr, int epilogue, int math, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(A && W && C, "omt_linear: null pointer");
  OMT_REQUIRE(M >= 0 && N > 0 && K > 0, "omt_linear: bad shape M=%d N=%d K=%d", M, N, K);
  OMT_REQUIRE(K % 8 == 0 && lda % 4 == 0 && ldc % 4 == 0 && N % 4 == 0, "omt_linear: K %% 8, lda/ldc/N %% 4 required (K=%d lda=%d ldc=%d N=%d)", K, lda, ldc, N);
  OMT_REQUIRE(epilogue == OMT_EPI_NONE || epilogue == OMT_EPI_GEGLU || epilogue == OMT_EPI_QKV, "omt_linear: unknown epilogue %d", epilogue);
  OMT_REQUIRE(!(epilogue == OMT_EPI_GEGLU && residual), "omt_linear: GEGLU epilogue takes no residual");
  OMT_REQUIRE(residual == nullptr || ldr % 4 == 0, "omt_linear: ldr %% 4 required");
  OMT_REQUIRE(((uintptr_t)A | (uintptr_t)W | (uintptr_t)C | (uintptr_t)bias | (uintptr_t)residual) % 16 == 0,
              "omt_linear: pointers must be 16-byte aligned");
  if (M == 0) return OMT_OK;
  OMT_REQUIRE(A2 == nullptr || (n_split > 0 && n_split % 128 == 0 && (uintptr_t)A2 % 16 == 0), "omt_linear2: bad n_split / A2");
  GemmArgs g{A, lda, a_seg, a_seg_stride, a_seg_off, W, C, ldc, c_seg, c_seg_stride, c_seg_off,
             M, N, K, bias, residual, ldr, A2, n_split, nullptr, nullptr, nullptr, nullptr, 0, 1};
  if (qk != nullptr) {
    g.rope_cos = qk->cos; g.rope_sin = qk->sin; g.q_scale = qk->q_scale; g.k_scale = qk->k_scale;
    g.qk_cols = qk->qk_cols; g.tokens = qk->tokens;
  }
  if (math == OMT_MATH_FP32) return launch_gemm_fp32(g, epilogue == OMT_EPI_QKV ? OMT_EPI_NONE : epilogue, (cudaStream_t)stream);
  if (math == OMT_MATH_3XTF32) {
    OMT_REQUIRE(W_lo != nullptr, "omt_linear: 3xTF32 needs W_lo");
    return launch_gemm_tc2(g, W_lo, epilogue, (cudaStream_t)stream, A2, n_split);
  }
  OMT_REQUIRE(math != OMT_MATH_F16X3, "omt_linear: the f16x3 path takes operand planes (omt_linear_h)");
  set_error("omt_linear: unknown math mode %d", math);
  return OMT_E_ARG;
}

extern "C" int omt_linear(const float* A, int lda, int a_seg, int a_seg_stride, int a_seg_off,
                          const float* W, const float* W_lo, float* C, int ldc, int c_seg, int c_seg_stride,
                          int c_seg_off, int M, int N, int K, const float* bias, const float* residual,
                          int ldr, int epilogue, int math, omt_stream_t stream) {
  return linear_impl(nullptr, A, nullptr, 0, lda, a_seg, a_seg_stride, a_seg_off, W, W_lo, C, ldc, c_seg, c_seg_stride, c_seg_off,
                     M, N, K, bias, residual, ldr, epilogue, math, stream);
}

extern "C" int omt_linear2(const float* A1, const float* A2, int n_split, int lda, const float* W, const float* W_lo,
                           float* C, int ldc, int M, int N, int K, int math, const float* q_scale,
                           const float* k_scale, const float* rope_cos, const float* rope_sin, int qk_cols, int tokens,
                           omt_stream_t stream) {
  if (q_scale == nullptr)
    return linear_impl(nullptr, A1, A2, n_split, lda, 0, 0, 0, W, W_lo, C, ldc, 0, 0, 0, M, N, K, nullptr, nullptr, 0,
                       OMT_EPI_NONE, math, stream);
  OMT_REQUIRE(k_scale != nullptr && qk_cols > 0 && qk_cols % 128 == 0 && qk_cols <= N && tokens > 0,
              "omt_linear2: bad q/k preparation arguments");
  OMT_REQUIRE((rope_cos == nullptr) == (rope_sin == nullptr), "omt_linear2: cos/sin must both be given");
  QkPrep qk{q_scale, k_scale, rope_cos, rope_sin, qk_cols, tokens};
  const bool fused = math == OMT_MATH_3XTF32;   // the wgmma 3xTF32 kernel applies rope + l2norm + scale in its epilogue
  int rc = linear_impl(&qk, A1, A2, n_split, lda, 0, 0, 0, W, W_lo, C, ldc, 0, 0, 0, M, N, K, nullptr, nullptr, 0,
                       fused ? OMT_EPI_QKV : OMT_EPI_NONE, math, stream);
  if (rc != OMT_OK || fused) return rc;
  // kernels without the fused epilogue (fp32): same arithmetic as a separate pass over q and k
  return omt_qk_prep(C, ldc, C + qk_cols / 2, ldc, q_scale, k_scale, rope_cos, rope_sin, M, tokens, qk_cols / 2 / 64, stream);
}
