// Attention v3: spatial (full, non-causal) attention core on sm_90a wgmma with 3xTF32 compensation.
//   O = softmax(scale * Q K^T) V  per (sequence, head), head dim 64, N % 128 == 0
//   (F.scaled_dot_product_attention at modules/attention.py:451).
//
// One CTA = two warpgroups, 64 query rows each; S and O live in registers (online softmax).  Every operand is split into
// tf32 hi / lo in shared memory by the CTA (Q once, K in place per key tile, V transposed into the K-major V^T tile the
// tf32 wgmma needs as its B operand), and every product takes three tf32 wgmmas (lo.hi + hi.lo + hi.hi).  P goes through a
// per-warpgroup shared-memory tile (tf32 hi / lo) as the A operand of the P.V wgmmas.
//   smem: Q_hi | Q_lo (32 KiB each) | K_hi | K_lo | V_raw | V^T_hi | V^T_lo (16 KiB each) | P[2 warpgroups] x (hi | lo) (16 KiB each)
// Every fp32 tile is stored as 32-column halves of 128-byte rows (SWIZZLE_128B, the layout the TMA lands).
#include "omt_common.cuh"
#include "tc_ptx.cuh"
#include <cuda.h>

namespace omt {
namespace atc3 {
using namespace omt::ptx;

constexpr int QT = 128, KT = 64, D = 64;
constexpr int HALF = 64 * 32 * 4;       // 8 KiB: 64 rows x 32 fp32 (one TMA box)
constexpr int Q_BYTES = QT * D * 4;     // 32 KiB: [column half][128 rows]
constexpr int K_BYTES = KT * D * 4;     // 16 KiB: [column half][64 rows]
constexpr int OFF_QH = 0, OFF_QL = Q_BYTES;
constexpr int OFF_KH = 2 * Q_BYTES, OFF_KL = OFF_KH + K_BYTES, OFF_VR = OFF_KL + K_BYTES;
constexpr int OFF_VH = OFF_VR + K_BYTES, OFF_VL = OFF_VH + K_BYTES;
constexpr int OFF_P = OFF_VL + K_BYTES;                              // [2 warpgroups] x (hi | lo), [key half][64 rows] each
constexpr int OFF_CTRL = OFF_P + 4 * K_BYTES;
constexpr int SMEM = OFF_CTRL + 64 + 1024;                           // barriers + alignment slack
constexpr int THREADS = 256;

struct Args {
  float* o; int ldo;
  uint16_t* o_hi; uint16_t* o_lo;   // optional operand planes instead of o
  int N;
  float scale_log2;
};

__device__ __forceinline__ void split_inplace(float4* h, float4* l, int idx) {
  const float4 v = h[idx];
  float4 hi, lo;
  hi.x = tf32_rn(v.x); hi.y = tf32_rn(v.y); hi.z = tf32_rn(v.z); hi.w = tf32_rn(v.w);
  lo.x = v.x - hi.x; lo.y = v.y - hi.y; lo.z = v.z - hi.z; lo.w = v.w - hi.w;
  h[idx] = hi;
  l[idx] = lo;
}
// byte offset of element (row, col) of a [col half][rows] SWIZZLE_128B fp32 tile (half_bytes apart)
__device__ __forceinline__ uint32_t sw_off(int row, int col, int half_bytes) {
  return (uint32_t)((col >> 5) * half_bytes + row * 128 + ((((col & 31) >> 2) ^ (row & 7)) << 4) + (col & 3) * 4);
}

__global__ void __launch_bounds__(THREADS, 1)
attn_tc3_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const Args a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_CTRL);
  uint64_t& q_full = bars[0];
  uint64_t& kv_full = bars[1];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2, qd = lane & 3;
  const int qt = blockIdx.x, head = blockIdx.y, seq = blockIdx.z;
  const int ntiles = a.N / KT;
  const int row_q0 = seq * a.N + qt * QT;
  const int row_k0 = seq * a.N;
  const int col0 = head * D;

  if (tid == 0) {
    prefetch_map(&tmQ); prefetch_map(&tmK); prefetch_map(&tmV);
    mbar_init(&q_full, 1); mbar_init(&kv_full, 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_sync();

  auto issue_kv = [&](int j) {
    const int kr = row_k0 + j * KT;
    mbar_expect_tx(&kv_full, 2 * K_BYTES);
    for (int c = 0; c < 2; ++c) {
      tma_load_2d(&tmK, &kv_full, smem + OFF_KH + c * HALF, col0 + 32 * c, kr);
      tma_load_2d(&tmV, &kv_full, smem + OFF_VR + c * HALF, col0 + 32 * c, kr);
    }
  };
  if (tid == 0) {
    mbar_expect_tx(&q_full, Q_BYTES);
    for (int c = 0; c < 2; ++c)
      for (int w = 0; w < 2; ++w) tma_load_2d(&tmQ, &q_full, smem + OFF_QH + c * (Q_BYTES / 2) + w * HALF, col0 + 32 * c, row_q0 + 64 * w);
    issue_kv(0);
  }
  // ---- Q: tf32 hi (in place) / lo
  mbar_wait(&q_full, 0);
#pragma unroll
  for (int i = 0; i < Q_BYTES / 16 / THREADS; ++i)
    split_inplace(reinterpret_cast<float4*>(smem + OFF_QH), reinterpret_cast<float4*>(smem + OFF_QL), tid + i * THREADS);

  const uint32_t sb = smem_u32(smem);
  const uint32_t p_hi = sb + OFF_P + wg * 2 * K_BYTES, p_lo = p_hi + K_BYTES;
  const int rl0 = (warp & 3) * 16 + (lane >> 2);   // this thread's rows (rl0, rl0 + 8) inside the warpgroup's 64
  float o_acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o_acc[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

  for (int j = 0; j < ntiles; ++j) {
    mbar_wait(&kv_full, j & 1);
    // ---- K split in place, V transposed into V^T [dim][key] and split
#pragma unroll
    for (int i = 0; i < K_BYTES / 16 / THREADS; ++i)
      split_inplace(reinterpret_cast<float4*>(smem + OFF_KH), reinterpret_cast<float4*>(smem + OFF_KL), tid + i * THREADS);
#pragma unroll
    for (int it = 0; it < K_BYTES / 16 / THREADS; ++it) {
      const int idx = it * THREADS + tid;
      const int key = idx & 63, d4 = idx >> 6;
      const float4 v = *reinterpret_cast<const float4*>(smem + OFF_VR + sw_off(key, d4 * 4, HALF));
      const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint32_t off = sw_off(d4 * 4 + i, key, HALF);
        const float hi = tf32_rn(e[i]);
        *reinterpret_cast<float*>(smem + OFF_VH + off) = hi;
        *reinterpret_cast<float*>(smem + OFF_VL + off) = e[i] - hi;
      }
    }
    fence_async_smem();
    __syncthreads();                               // split tiles (and, on the first tile, Q) are complete
    // ---- S = Q K^T
    float sv[32];
    wg_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {               // 8 tf32 of the head dim per MMA
      const uint32_t qo = (kk >> 2) * (Q_BYTES / 2) + wg * HALF + (kk & 3) * 32;
      const uint32_t ko = (kk >> 2) * HALF + (kk & 3) * 32;
      wgmma_tf32_n64(sv, desc_sw128(sb + OFF_QL + qo), desc_sw128(sb + OFF_KH + ko), kk != 0);
      wgmma_tf32_n64(sv, desc_sw128(sb + OFF_QH + qo), desc_sw128(sb + OFF_KL + ko), 1);
      wgmma_tf32_n64(sv, desc_sw128(sb + OFF_QH + qo), desc_sw128(sb + OFF_KH + ko), 1);
    }
    wg_commit();
    wg_wait<0>();
    // ---- online softmax: a row's 64 keys sit in the 4 lanes of a quad (16 each)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) mx = fmaxf(mx, fmaxf(sv[4 * jj + 2 * h], sv[4 * jj + 2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[h], mx);
      const float alpha = exp2f((m_run[h] - m_new) * a.scale_log2);
      m_run[h] = m_new;
      const int r = rl0 + 8 * h;
      float psum = 0.f;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const int key = 8 * jj + 2 * qd;
        const float e0 = exp2f((sv[4 * jj + 2 * h] - m_new) * a.scale_log2);
        const float e1 = exp2f((sv[4 * jj + 2 * h + 1] - m_new) * a.scale_log2);
        psum += e0 + e1;
        const float h0 = tf32_rn(e0), h1 = tf32_rn(e1);
        const uint32_t off = sw_off(r, key, K_BYTES / 2);
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(p_hi + off), "f"(h0), "f"(h1) : "memory");
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(p_lo + off), "f"(e0 - h0), "f"(e1 - h1) : "memory");
        o_acc[4 * jj + 2 * h] *= alpha;
        o_acc[4 * jj + 2 * h + 1] *= alpha;
      }
      l_run[h] = l_run[h] * alpha + psum;          // partial row sum over this lane's keys
    }
    fence_async_smem();
    wg_bar(1 + wg);
    // ---- O += P V
    wg_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {               // 8 keys per MMA
      const uint32_t ko = (kk >> 2) * (K_BYTES / 2) + (kk & 3) * 32;
      wgmma_tf32_n64(o_acc, desc_sw128(p_lo + ko), desc_sw128(sb + OFF_VH + ko), 1);
      wgmma_tf32_n64(o_acc, desc_sw128(p_hi + ko), desc_sw128(sb + OFF_VL + ko), 1);
      wgmma_tf32_n64(o_acc, desc_sw128(p_hi + ko), desc_sw128(sb + OFF_VH + ko), 1);
    }
    wg_commit();
    wg_wait<0>();
    __syncthreads();                               // every K / V / P tile of this key tile has been read
    if (tid == 0 && j + 1 < ntiles) issue_kv(j + 1);
  }
  // total row sum over the quad
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_run[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = 1.0f / l;
    const size_t ooff = (size_t)(row_q0 + wg * 64 + rl0 + 8 * h) * a.ldo + col0 + 2 * qd;
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const float2 ov = make_float2(o_acc[4 * jj + 2 * h] * inv, o_acc[4 * jj + 2 * h + 1] * inv);
      if (a.o_hi != nullptr) store_split2(a.o_hi, a.o_lo, ooff + 8 * jj, ov);
      else *reinterpret_cast<float2*>(a.o + ooff + 8 * jj) = ov;
    }
  }
}

static int encode2d(CUtensorMap* m, const float* base, int cols, long long rows, int ld, int box_rows) {
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
  cuuint32_t box[2] = {32, (cuuint32_t)box_rows};
  return encode_tiled(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, base, 2, dims, strides, box);
}

}  // namespace atc3

int launch_attn_tc3(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, float* o, uint16_t* o_hi,
                    uint16_t* o_lo, int ldo, int n_seq, int N, int heads, float scale, cudaStream_t st) {
  using namespace atc3;
  CUtensorMap tmQ, tmK, tmV;
  const long long rows = (long long)n_seq * N;
  int rc = encode2d(&tmQ, q, heads * D, rows, ldq, 64);
  if (rc) return rc;
  rc = encode2d(&tmK, k, heads * D, rows, ldk, KT);
  if (rc) return rc;
  rc = encode2d(&tmV, v, heads * D, rows, ldv, KT);
  if (rc) return rc;
  static KernelSetup setup;
  if ((rc = setup.smem(attn_tc3_kernel, SMEM))) return rc;
  Args a{o, ldo, o_hi, o_lo, N, scale * 1.4426950408889634f};
  dim3 grid(N / QT, heads, n_seq);
  OMT_CUDA(launch_k(attn_tc3_kernel, grid, dim3(THREADS), SMEM, st, tmQ, tmK, tmV, a));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

}  // namespace omt
