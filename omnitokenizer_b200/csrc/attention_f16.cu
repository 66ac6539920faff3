// Attention v4: spatial (full, non-causal) attention core on sm_90a wgmma (f16) with row-scaled fp16 operand planes.
//   O = softmax(scale * Q K^T) V  per (sequence, head), head dim 64, N % 128 == 0
//   (F.scaled_dot_product_attention at modules/attention.py:451).
//
// Operands come from the QKV GEMM epilogue (gemm_wgmma.cuh, OMT_EPI_QKV_PLANES) already in tensor-core form:
//   q, k : after rope + l2norm + per-dim scale every component is bounded by max|q_scale| / max|k_scale|, so ONE static
//          power of two per layer puts them in fp16 range: planes hi = fp16(x * 2^e), lo = fp16(x * 2^e - hi)
//   v    : unbounded, scaled per (row, head); the inverse scales live in vinv[head][row]
// so S = Q K^T and O_j = P_j V_j each take THREE f16 wgmmas per 16-deep k-step into ONE fp32 accumulator
// (hi.hi + hi.lo + lo.hi).
//   * Q, K and V tiles come straight from TMA; V is consumed as an MN-MAJOR B operand (the token-major [64 keys][64 dims]
//     tile the TMA lands is the canonical SWIZZLE_128B MN-major layout), so nothing is transposed anywhere.
//   * the per-key inverse V scale is folded into P: P'' = p * vinv_j * 2^ep with ONE power of two per CTA taken from the
//     largest vinv of the sequence, so p'' stays in fp16 range; 2^-ep comes off with the final 1 / row-sum.
// One CTA = two warpgroups, 64 query rows each (S and O in registers, online softmax); P'' goes through a per-warpgroup
// shared-memory tile as the A operand of the P.V wgmmas.  K / V tiles are double-buffered; thread 0 issues the TMA loads.
#include "omt_common.cuh"
#include "tc_ptx.cuh"
#include <cuda.h>

namespace omt {
int g_attn_f16_ctas = 2;      // omt_set_option("attn_f16_ctas", 1 | 2): accepted for compatibility (one kernel shape on sm_90)
namespace af16 {
using namespace omt::ptx;

constexpr int QT = 128, KT = 64, D = 64;
constexpr int TILE = KT * D * 2;                    // 8 KiB: one 64 x 64 fp16 plane tile
constexpr int OFF_Q = 0;                            // Q_hi [2 warpgroups] | Q_lo [2]
constexpr int OFF_KV = 4 * TILE;                    // [2 stages] x (K_hi | K_lo | V_hi | V_lo)
constexpr int OFF_P = OFF_KV + 8 * TILE;            // [2 warpgroups] x (P_hi | P_lo)
constexpr int OFF_CTRL = OFF_P + 4 * TILE;
constexpr int SMEM = OFF_CTRL + 1024 + 1024;        // barriers / reduction + alignment slack
constexpr int THREADS = 256;

struct Args {
  const float* vinv;                                       // [heads][rows] inverse scales of the v rows
  long long rows;                                          // n_seq * N
  float* o; uint16_t* o_hi; uint16_t* o_lo; int ldo;
  int N;
  float scale_log2;                                        // scale * log2(e) / (q plane scale * k plane scale)
};

__global__ void __launch_bounds__(THREADS, 1)
attn_f16_kernel(const __grid_constant__ CUtensorMap tmQh, const __grid_constant__ CUtensorMap tmQl,
                const __grid_constant__ CUtensorMap tmKh, const __grid_constant__ CUtensorMap tmKl,
                const __grid_constant__ CUtensorMap tmVh, const __grid_constant__ CUtensorMap tmVl, const Args a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_CTRL);
  uint64_t& q_full = bars[0];
  uint64_t* full = bars + 1;                                          // [2] K / V planes of a key tile landed
  float* red = reinterpret_cast<float*>(smem + OFF_CTRL + 64);        // [8] per-warp maxima of vinv

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2, qd = lane & 3;
  const int qt = blockIdx.x, head = blockIdx.y, seq = blockIdx.z;
  const int ntiles = a.N / KT;
  const int row_q0 = seq * a.N + qt * QT;
  const int row_k0 = seq * a.N;
  const int col0 = head * D;

  if (tid == 0) {
    prefetch_map(&tmQh); prefetch_map(&tmQl); prefetch_map(&tmKh); prefetch_map(&tmKl); prefetch_map(&tmVh); prefetch_map(&tmVl);
    mbar_init(&q_full, 1); mbar_init(&full[0], 1); mbar_init(&full[1], 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_sync();

  auto issue_kv = [&](int j) {
    const int s = j & 1;
    uint8_t* sp = smem + OFF_KV + s * 4 * TILE;
    const int kr = row_k0 + j * KT;
    mbar_expect_tx(&full[s], 4 * TILE);
    tma_load_2d(&tmKh, &full[s], sp, col0, kr);
    tma_load_2d(&tmKl, &full[s], sp + TILE, col0, kr);
    tma_load_2d(&tmVh, &full[s], sp + 2 * TILE, col0, kr);
    tma_load_2d(&tmVl, &full[s], sp + 3 * TILE, col0, kr);
  };
  if (tid == 0) {
    mbar_expect_tx(&q_full, 4 * TILE);
    for (int w = 0; w < 2; ++w) {
      tma_load_2d(&tmQh, &q_full, smem + OFF_Q + w * TILE, col0, row_q0 + w * 64);
      tma_load_2d(&tmQl, &q_full, smem + OFF_Q + (2 + w) * TILE, col0, row_q0 + w * 64);
    }
    issue_kv(0);
    if (ntiles > 1) issue_kv(1);
  }

  // ---- one power of two for P'' = p * vinv_j: the largest inverse V scale of this sequence and head
  const float* vinv_h = a.vinv + (size_t)head * a.rows + row_k0;
  float vmx = 0.f;
  for (int i = tid; i < a.N; i += THREADS) vmx = fmaxf(vmx, __ldg(vinv_h + i));
  vmx = warp_max(vmx);
  if (lane == 0) red[warp] = vmx;
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 8; ++i) vmx = fmaxf(vmx, red[i]);
  float p_scale, p_inv;
  row_scale(vmx, p_scale, p_inv);                  // p * vinv_j * p_scale <= 2^15 for every key (p <= 1)

  const uint32_t sb = smem_u32(smem);
  const uint64_t dq_hi = desc_sw128(sb + OFF_Q + wg * TILE), dq_lo = desc_sw128(sb + OFF_Q + (2 + wg) * TILE);
  const uint32_t p_hi = sb + OFF_P + wg * 2 * TILE, p_lo = p_hi + TILE;
  const uint64_t dp_hi = desc_sw128(p_hi), dp_lo = desc_sw128(p_lo);
  const int rl0 = (warp & 3) * 16 + (lane >> 2);   // this thread's rows (rl0, rl0 + 8) inside the warpgroup's 64
  float o_acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o_acc[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  mbar_wait(&q_full, 0);

  for (int j = 0; j < ntiles; ++j) {
    const int s = j & 1;
    const uint32_t kv = sb + OFF_KV + s * 4 * TILE;
    mbar_wait(&full[s], (j >> 1) & 1);
    float sv[32];
    {
      const uint64_t dk_hi = desc_sw128(kv), dk_lo = desc_sw128(kv + TILE);
      wg_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {             // 16 of the 64 head dims per MMA
        const uint64_t adv = (uint64_t)(kk * 2);
        wgmma_f16_n64(sv, dq_lo + adv, dk_hi + adv, kk != 0);
        wgmma_f16_n64(sv, dq_hi + adv, dk_lo + adv, 1);
        wgmma_f16_n64(sv, dq_hi + adv, dk_hi + adv, 1);
      }
      wg_commit();
      wg_wait<0>();
    }
    // online softmax over this tile: a row's 64 keys sit in the 4 lanes of a quad (16 each)
    float alpha[2], nm[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) mx = fmaxf(mx, fmaxf(sv[4 * jj + 2 * h], sv[4 * jj + 2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[h], mx);
      alpha[h] = ex2_fast((m_run[h] - m_new) * a.scale_log2);
      m_run[h] = m_new;
      nm[h] = -m_new;
    }
    const float* vi = vinv_h + j * KT;
    float ps[2] = {0.f, 0.f};
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const int key = 8 * jj + 2 * qd;
      const float2 w = __ldg(reinterpret_cast<const float2*>(vi + key));
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float e0 = ex2_fast((sv[4 * jj + 2 * h] + nm[h]) * a.scale_log2);      // the row maximum maps to exactly 1
        const float e1 = ex2_fast((sv[4 * jj + 2 * h + 1] + nm[h]) * a.scale_log2);
        ps[h] += e0 + e1;
        uint32_t hw, lw;
        split2u(e0 * (w.x * p_scale), e1 * (w.y * p_scale), hw, lw);
        const int r = rl0 + 8 * h;
        const uint32_t off = (uint32_t)r * 128u + (uint32_t)((jj ^ (r & 7)) << 4) + (uint32_t)(qd * 4);
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(p_hi + off), "r"(hw) : "memory");
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(p_lo + off), "r"(lw) : "memory");
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      l_run[h] = fmaf(l_run[h], alpha[h], ps[h]);  // partial row sum over this lane's keys
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) { o_acc[4 * jj + 2 * h] *= alpha[h]; o_acc[4 * jj + 2 * h + 1] *= alpha[h]; }
    }
    fence_async_smem();
    wg_bar(1 + wg);
    {
      const uint32_t vh = kv + 2 * TILE, vl = kv + 3 * TILE;
      wg_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {             // 16 keys per MMA: 16 rows of the MN-major V tile = 2 KiB
        const uint64_t adv = (uint64_t)(kk * 2);
        const uint64_t dvh = desc_sw128(vh + kk * 2048), dvl = desc_sw128(vl + kk * 2048);
        wgmma_f16_n64_tb(o_acc, dp_lo + adv, dvh, 1);
        wgmma_f16_n64_tb(o_acc, dp_hi + adv, dvl, 1);
        wgmma_f16_n64_tb(o_acc, dp_hi + adv, dvh, 1);
      }
      wg_commit();
      wg_wait<0>();
    }
    __syncthreads();                               // both warpgroups are done with K / V stage s and their P tiles
    if (tid == 0 && j + 2 < ntiles) issue_kv(j + 2);
  }
  // total row sum over the quad; 2^-ep undoes the P'' scale
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_run[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = p_inv / l;
    const size_t ooff = (size_t)(row_q0 + wg * 64 + rl0 + 8 * h) * a.ldo + col0 + 2 * qd;
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const float2 ov = make_float2(o_acc[4 * jj + 2 * h] * inv, o_acc[4 * jj + 2 * h + 1] * inv);
      if (a.o_hi != nullptr) store_split2(a.o_hi, a.o_lo, ooff + 8 * jj, ov);
      else *reinterpret_cast<float2*>(a.o + ooff + 8 * jj) = ov;
    }
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static int encode2d(CUtensorMap* m, const uint16_t* base, int cols, long long rows, int ld) {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  if (fn == nullptr) { set_error("cuTensorMapEncodeTiled entry point not found"); return OMT_E_CUDA; }
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)KT};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<uint16_t*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d)", (int)r); return OMT_E_CUDA; }
  return OMT_OK;
}

}  // namespace af16
}  // namespace omt

using namespace omt;

extern "C" int omt_attn_spatial_h(const uint16_t* q_hi, const uint16_t* q_lo, int ldq, const uint16_t* k_hi,
                                  const uint16_t* k_lo, int ldk, const uint16_t* v_hi, const uint16_t* v_lo, int ldv,
                                  const float* vinv, float qk_plane_scale, float* o, uint16_t* o_hi, uint16_t* o_lo, int ldo,
                                  int n_seq, int N, int heads, float scale, omt_stream_t stream) {
  using namespace af16;
  OMT_ENTER();
  OMT_REQUIRE(q_hi && q_lo && k_hi && k_lo && v_hi && v_lo && vinv && (o || o_hi) && ((o_hi == nullptr) == (o_lo == nullptr)),
              "omt_attn_spatial_h: null pointer");
  OMT_REQUIRE(N > 0 && N % QT == 0, "omt_attn_spatial_h: N=%d must be a multiple of 128", N);
  OMT_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 4 == 0, "omt_attn_spatial_h: bad leading dims");
  OMT_REQUIRE(((uintptr_t)q_hi | (uintptr_t)q_lo | (uintptr_t)k_hi | (uintptr_t)k_lo | (uintptr_t)v_hi | (uintptr_t)v_lo | (uintptr_t)vinv |
               (uintptr_t)o | (uintptr_t)o_hi | (uintptr_t)o_lo) % 16 == 0, "omt_attn_spatial_h: pointers must be 16-byte aligned");
  OMT_REQUIRE(heads > 0 && heads <= 65535 && n_seq <= 65535 && qk_plane_scale > 0.f, "omt_attn_spatial_h: bad arguments");
  if (n_seq == 0) return OMT_OK;
  const long long rows = (long long)n_seq * N;
  CUtensorMap tmQh, tmQl, tmKh, tmKl, tmVh, tmVl;
  int rc;
  if ((rc = encode2d(&tmQh, q_hi, heads * D, rows, ldq))) return rc;
  if ((rc = encode2d(&tmQl, q_lo, heads * D, rows, ldq))) return rc;
  if ((rc = encode2d(&tmKh, k_hi, heads * D, rows, ldk))) return rc;
  if ((rc = encode2d(&tmKl, k_lo, heads * D, rows, ldk))) return rc;
  if ((rc = encode2d(&tmVh, v_hi, heads * D, rows, ldv))) return rc;
  if ((rc = encode2d(&tmVl, v_lo, heads * D, rows, ldv))) return rc;
  static bool attr[64];
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev >= 0 && dev < 64 && !attr[dev]) {
    OMT_CUDA(cudaFuncSetAttribute(attn_f16_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    attr[dev] = true;
  }
  Args a{vinv, rows, o, o_hi, o_lo, ldo, N, scale * 1.4426950408889634f / qk_plane_scale};
  dim3 grid(N / QT, heads, n_seq);
  OMT_CUDA(launch_k(attn_f16_kernel, grid, dim3(THREADS), SMEM, (cudaStream_t)stream, tmQh, tmQl, tmKh, tmKl, tmVh, tmVl, a));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}
