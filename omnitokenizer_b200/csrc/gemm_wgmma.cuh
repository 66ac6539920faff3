// The tensor-core GEMM of both error-compensated paths, on sm_90a wgmma:
//
//   C[M,N] = A[M,K] . W[N,K]^T (+bias)(+residual) | GEGLU | rope+l2norm+scale,   fp32-grade accuracy.
//
//   TF32 = true  (3xTF32, gemm_tc2.cu): A arrives as fp32 and is split into tf32 hi / lo in shared memory by the warpgroup
//                that consumes it; W arrives pre-split (hi = tf32(W), lo = W - hi).  A.W ~= A_lo.W_hi + A_hi.W_lo + A_hi.W_hi.
//   TF32 = false (f16x3, gemm_f16.cu): A and W arrive as fp16 hi / lo planes written by their producers (omt_common.cuh).
//                NACC = 2: lo planes carry 2^11, the cross products go to a second accumulator folded in as main + cross * 2^-11;
//                NACC = 1: row-scaled planes, all three products share one accumulator, the epilogue multiplies by the exact
//                inverse scales (a_rs[row] * w_scale).
//   H1 = true   (f16x1, gemm_f16.cu omt_linear_h1): the throughput form.  A stage holds only A_hi and W_hi and each
//                16-deep k-step issues ONE wgmma per 64-row half into the single accumulator; the epilogue applies the same
//                row-scaled factor (the 2^11 form launches with both factors 1) and writes only the hi planes.
//
// Warp-specialised and persistent:
//   * one producer warpgroup (one thread) issues every TMA load; two consumer warpgroups hold the accumulators in
//     registers.  setmaxnreg moves registers from the producer to the consumers.
//   * every 128-byte k-block of the operands lands by TMA (SWIZZLE_128B, the canonical K-major wgmma layout) in one of
//     STAGES stages of a full / empty mbarrier ring.  A consumer keeps one wgmma group in flight and releases a stage once
//     the wgmmas that read it have retired, so the producer refills it while the next k-block computes.
//   * the grid is as many CTAs as are resident; each walks the tiles (n fastest) with a static stride, and the producer
//     runs ahead into the next tile while the consumers run the epilogue.
// Two consumer schedules, fixed by the template arguments:
//   * ping-pong (TF32 == false, NACC == 1): each consumer warpgroup owns whole 128 x 128 tiles (128 accumulators a
//     thread), warpgroup 1 the even tiles of the CTA's walk and warpgroup 2 the odd ones.  An ordering barrier lets a
//     warpgroup issue a tile's wgmmas only once the other one has issued its last k-block, so one warpgroup's epilogue
//     runs while the other keeps the tensor pipe busy.
//   * cooperative (NACC == 2, whose two accumulators would need 256 registers for 128 rows, and TF32, whose warpgroups
//     split their own 64 rows of A in shared memory): both warpgroups compute every tile, 64 rows each, and run the
//     epilogue together.
// Both issue the same products in the same k order for every output element, so they give the same bits.
// The epilogue works on the accumulator fragments in place: a row's 64-column head is spread over the 4 lanes of a quad,
// so the l2 norm and the v-plane maximum are two-step shuffles.  The f16 epilogues that write operand planes (GEGLU: a
// quad holds only 8 bytes of a U-plane row; QKV planes: 16 bytes of a head's row) stage 64 rows x 64 columns of the hi /
// lo planes at a time in shared memory, and one thread of the warpgroup writes them out by TMA stores.
#pragma once
#include "omt_common.cuh"
#include "tc_ptx.cuh"
#include <cuda.h>

namespace omt {
namespace wgg {
using namespace omt::ptx;

constexpr int BM = 128, BN = 128;
constexpr int THREADS = 384;                  // warpgroup 0: producer; 1, 2: consumers
constexpr int ORDER_BAR = 3;                  // ping-pong: named barriers 3, 4 ("consumer 0 / 1 may issue"); 1, 2 are wg_bar
constexpr int STAGE_BYTES = 4 * 16384;        // A (hi), A_lo, W_hi, W_lo: 128 rows x 128 bytes each
constexpr int STAGES = 3;
// H1: a stage is A_hi | W_hi, half the bytes, so the ring holds twice as many 128-byte k-slabs in the same shared memory
template <bool H1> __host__ __device__ constexpr int stage_bytes() { return H1 ? 2 * 16384 : STAGE_BYTES; }
template <bool H1> __host__ __device__ constexpr int stages() { return H1 ? 2 * STAGES : STAGES; }
// f16 plane-writing epilogues (GEGLU, QKV planes): per consumer warpgroup, 64 rows x 64 columns of the hi and lo planes
// (the U planes of one 64-row half, or one head of one) staged in shared memory in the SWIZZLE_128B layout of a TMA box,
// so that they leave by TMA stores.  Only those instantiations reserve it: the others keep the larger L1.  The f16x1 QKV
// planes epilogue stores its hi plane from the fragments: behind its single-product mainloop, the per-head hand-off of
// the stage between the warpgroup and the TMA store measured slower than the per-thread stores.
constexpr int EPI_STAGE_BYTES = 2 * 64 * 128;
template <bool TF32, int EPI, bool H1>
__host__ __device__ constexpr bool tma_planes() {
  return !TF32 && (EPI == OMT_EPI_GEGLU || (EPI == OMT_EPI_QKV_PLANES && !H1));
}
template <bool TF32, int EPI, bool H1 = false>
constexpr int smem_bytes() { return stages<H1>() * stage_bytes<H1>() + (tma_planes<TF32, EPI, H1>() ? 2 * EPI_STAGE_BYTES : 0) + 1024; }
// __launch_bounds__(384, 1) caps the kernel at 168 registers a thread: 40 * 128 + 232 * 256 == 168 * 384
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;

struct Args {
  int M, N, K;
  int num_m_blk, n_split;
  int a_seg, a_seg_stride, a_seg_off;         // A row map (the TMA strides live in the tensor maps; the epilogue needs it for a_rs)
  const float* a_rs; const float* a2_rs;      // NACC == 1: inverse row scales of the A planes (second: dual-A columns >= n_split)
  float a_rs_uniform;                         // NACC == 1 with a_rs == NULL: one inverse scale for every row
  float w_scale;                              // NACC == 1: inverse scale of the W planes
  float u_scale;                              // f16 GEGLU: > 0 -> U planes in the static-scaled form (unscaled lo), else 2^11-scaled lo
  float* c; int ldc;                          // fp32 output (plain / QKV; 3xTF32 GEGLU: C has N/2 columns)
  int c_seg, c_seg_stride, c_seg_off;         // C / residual row map
  const float* bias;
  const float* residual; int ldr;
  uint16_t* u_hi; uint16_t* u_lo; int ldu;    // f16 GEGLU: planes of U[M, N/2]; QKV_PLANES: planes of q | k | v [M, N]
  const float* rope_cos; const float* rope_sin; const float* q_scale; const float* k_scale;
  int qk_cols; int tokens;
  float q_ps, k_ps;                           // QKV_PLANES: static plane scales of the q and k heads (powers of two)
  float* vinv;                                // QKV_PLANES: [v heads][M] inverse per-(row, head) scale of the v planes
};

// One thread writes a warpgroup's staged planes (64 rows from `row`, 64 columns from `col`) by TMA, as two 32-row boxes
// per plane: a C row-map segment is a multiple of 32 rows, so no box crosses one.  Rows at or past M fall outside the
// map and are not written.
template <bool H1>
__device__ __forceinline__ void store_planes(const CUtensorMap* mh, const CUtensorMap* ml, const uint8_t* stage, int col,
                                             int row, int seg) {
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int r = row + 32 * i;
    const int c1 = seg > 0 ? r % seg : r, c2 = seg > 0 ? r / seg : 0;
    tma_store_3d(mh, stage + i * 32 * 128, col, c1, c2);
    if (!H1) tma_store_3d(ml, stage + 64 * 128 + i * 32 * 128, col, c1, c2);
  }
  bulk_commit();
}

// Epilogue of one 64-row half of a tile on a consumer warpgroup's fragments (rows [m0 + 64 half, +64), columns [n0, +128)).
// `stage` is the warpgroup's EPI_STAGE_BYTES of shared memory, `bar` its named barrier; tmUh / tmUl map the output planes
// of the plane-writing f16 epilogues.
template <bool TF32, int NACC, int EPI, bool H1>
__device__ __forceinline__ void epilogue(const Args& g, const float (&acc)[BN / 2], const float (&crs)[NACC == 2 ? BN / 2 : 1],
                                         int m0, int n0, bool second, int half, int warp, int lane, uint8_t* stage, int bar,
                                         const CUtensorMap* tmUh, const CUtensorMap* tmUl) {
  const int qd = lane & 3;                      // column pair 8 j + 2 qd inside every 8-column block
  const bool elected = (warp & 3) == 0 && lane == 0;   // the warpgroup's TMA-store thread
  int mrow[2];
  mrow[0] = m0 + half * 64 + (warp & 3) * 16 + (lane >> 2);
  mrow[1] = mrow[0] + 8;
  float v[2][BN / 4];                           // [row (+0 / +8)][2 j + e]: columns 8 j + 2 qd + e of the tile
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float os = 1.f;
    if (!TF32 && NACC == 1) {
      const float* rs = second ? g.a2_rs : g.a_rs;
      const int m = mrow[h];
      os = g.w_scale * (rs == nullptr ? g.a_rs_uniform : (m < g.M ? __ldg(rs + map_row(m, g.a_seg, g.a_seg_stride, g.a_seg_off)) : 1.0f));
    }
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int i = 4 * j + 2 * h + e;
        float x = acc[i];
        if constexpr (!TF32 && NACC == 2) x = fmaf(crs[i], 1.0f / F16X3_LO_SCALE, x);
        if (!TF32 && NACC == 1) x = x * os;
        v[h][2 * j + e] = x;
      }
  }

  if constexpr (EPI == OMT_EPI_QKV || EPI == OMT_EPI_QKV_PLANES) {
    constexpr bool STAGED = tma_planes<TF32, EPI, H1>();
#pragma unroll
    for (int hd = 0; hd < BN / 64; ++hd) {
      const int nh = n0 + hd * 64;              // first column of this head
      if (nh >= g.N) break;                     // warpgroup-uniform
      if constexpr (STAGED) {
        if (elected) bulk_wait_read<0>();       // the previous TMA store has read the stage
        wg_bar(bar);
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = mrow[h];
        float* x = &v[h][hd * 16];              // this lane's 16 values of the head: dims 8 j + 2 qd + e, j < 8
        if (nh < g.qk_cols) {
          // rope + l2norm + per-dim scale (attention.py:417-421, 435-437)
          if (g.rope_cos != nullptr) {
            const int pos = (m < g.M ? m : 0) % g.tokens;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int p = 4 * j + qd;         // complex pair (dims 2p, 2p + 1)
              const float cc = __ldg(g.rope_cos + (size_t)pos * 32 + p), ss = __ldg(g.rope_sin + (size_t)pos * 32 + p);
              const float a = x[2 * j], b = x[2 * j + 1];
              x[2 * j] = a * cc - b * ss;
              x[2 * j + 1] = a * ss + b * cc;
            }
          }
          float sq = 0.f;
#pragma unroll
          for (int i = 0; i < 16; ++i) sq = fmaf(x[i], x[i], sq);
          sq += __shfl_xor_sync(0xffffffffu, sq, 1);
          sq += __shfl_xor_sync(0xffffffffu, sq, 2);
          const float inv = 1.0f / fmaxf(sqrtf(sq), 1e-12f);
          const float* scv = (nh < g.qk_cols / 2) ? g.q_scale : g.k_scale;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float2 s2 = __ldg(reinterpret_cast<const float2*>(scv + 8 * j + 2 * qd));
            x[2 * j] = x[2 * j] * inv * s2.x;
            x[2 * j + 1] = x[2 * j + 1] * inv * s2.y;
          }
        }
        if constexpr (EPI == OMT_EPI_QKV) {
          if (m < g.M) {
            float* crow = g.c + map_row(m, g.c_seg, g.c_seg_stride, g.c_seg_off) * g.ldc + nh + 2 * qd;
#pragma unroll
            for (int j = 0; j < 8; ++j) *reinterpret_cast<float2*>(crow + 8 * j) = make_float2(x[2 * j], x[2 * j + 1]);
          }
        } else {
          // operand planes for the attention core: q / k with the layer's static power-of-two scale, v scaled per
          // (row, head) with the inverse scale kept in vinv
          float sc = nh < g.qk_cols / 2 ? g.q_ps : g.k_ps;
          if (nh >= g.qk_cols) {
            float mx = 0.f;
#pragma unroll
            for (int i = 0; i < 16; ++i) mx = fmaxf(mx, fabsf(x[i]));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            float inv;
            row_scale(mx, sc, inv);
            if (m < g.M && qd == 0) g.vinv[(size_t)((nh - g.qk_cols) >> 6) * g.M + m] = inv;
          }
          if constexpr (STAGED) {
            // the head's 64 columns of row r in the stage: 16-byte chunk j at chunk j ^ (r & 7) (the TMA box layout;
            // the 8 rows of a warp's store land in 8 different bank groups)
            const int r = (warp & 3) * 16 + (lane >> 2) + 8 * h;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              uint32_t hw, lw;
              split2u(x[2 * j] * sc, x[2 * j + 1] * sc, hw, lw);
              const int off = r * 128 + ((j ^ (r & 7)) << 4) + 4 * qd;
              *reinterpret_cast<uint32_t*>(stage + off) = hw;
              *reinterpret_cast<uint32_t*>(stage + 64 * 128 + off) = lw;
            }
          } else if (m < g.M) {
            const size_t off = (size_t)m * g.ldu + nh + 2 * qd;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              uint32_t hw, lw;
              split2u(x[2 * j] * sc, x[2 * j + 1] * sc, hw, lw);
              *reinterpret_cast<uint32_t*>(g.u_hi + off + 8 * j) = hw;
              if (!H1) *reinterpret_cast<uint32_t*>(g.u_lo + off + 8 * j) = lw;
            }
          }
        }
      }
      if constexpr (STAGED) {
        fence_async_smem();                     // this thread's stage writes -> visible to the TMA store
        wg_bar(bar);
        if (elected) store_planes<false>(tmUh, tmUl, stage, nh, m0 + half * 64, 0);
      }
    }
  } else if constexpr (EPI == OMT_EPI_GEGLU) {
    // packed columns (2i, 2i+1) = (value_i, gate_i): U[:, i] = gelu_erf(gate) * value; lanes qd and qd ^ 1 hold neighbouring
    // outputs.
    if constexpr (TF32) {
      // the even lane stores both
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = mrow[h];
        const long long prow = map_row(m < g.M ? m : 0, g.c_seg, g.c_seg_stride, g.c_seg_off);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int n = n0 + 8 * j + 2 * qd;
          float val = v[h][2 * j], gate = v[h][2 * j + 1];
          if (g.bias != nullptr && n < g.N) { val += __ldg(g.bias + n); gate += __ldg(g.bias + n + 1); }
          const float o = gelu_erf(gate) * val;
          const float o1 = __shfl_xor_sync(0xffffffffu, o, 1);
          if ((qd & 1) == 0 && m < g.M && n < g.N) *reinterpret_cast<float2*>(g.c + prow * g.ldc + (n >> 1)) = make_float2(o, o1);
        }
      }
    } else {
      // f16: the 64 x 64 U values of the half go to the planes in `stage` (row r at r * 128 bytes, its 16-byte chunk c
      // at chunk c ^ (r & 7): the 8 rows of a store land in 8 different bank groups), then one thread writes them out
      // by TMA stores.
      if constexpr (!H1) {
        // The pair of 8-column blocks (2k, 2k + 1) is split between the lanes of a pair: the even lane packs the U pair
        // of block 2k, the odd lane that of block 2k + 1, each after one exchange.  So every lane splits 8 pairs a row
        // and the four lanes of a quad fill one 16-byte chunk.  The whole half is packed before the warpgroup waits for
        // the stage, which the previous half's TMA store may still be reading.
        const bool odd = (qd & 1) != 0;
        uint32_t hw[2][BN / 16], lw[2][BN / 16];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int k = 0; k < BN / 16; ++k) {
            float o[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int j = 2 * k + e;
              const int n = n0 + 8 * j + 2 * qd;
              float val = v[h][2 * j], gate = v[h][2 * j + 1];
              if (g.bias != nullptr && n < g.N) { val += __ldg(g.bias + n); gate += __ldg(g.bias + n + 1); }
              o[e] = gelu_erf(gate) * val;
            }
            const float got = __shfl_xor_sync(0xffffffffu, odd ? o[0] : o[1], 1);   // the partner's o of my block
            const float a = odd ? got : o[0], b = odd ? o[1] : got;                  // U columns i, i + 1
            if (g.u_scale > 0.f) split2u(a * g.u_scale, b * g.u_scale, hw[h][k], lw[h][k]);
            else split2(a, b, hw[h][k], lw[h][k]);
          }
        }
        if (elected) bulk_wait_read<0>();     // the previous half's TMA store has read the stage
        wg_bar(bar);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = (warp & 3) * 16 + (lane >> 2) + 8 * h;
#pragma unroll
          for (int k = 0; k < BN / 16; ++k) {
            // U column (8 (2k + odd) + 2 (qd & ~1)) / 2: byte 16 k + 8 odd + 4 (qd >> 1) of the row
            const int off = r * 128 + ((k ^ (r & 7)) << 4) + 8 * (qd & 1) + 4 * (qd >> 1);
            *reinterpret_cast<uint32_t*>(stage + off) = hw[h][k];
            *reinterpret_cast<uint32_t*>(stage + 64 * 128 + off) = lw[h][k];
          }
        }
      } else {
        // f16x1 (hi plane only; the paired form spills here): the even lane packs both outputs of each block
        if (elected) bulk_wait_read<0>();     // the previous half's TMA store has read the stage
        wg_bar(bar);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = (warp & 3) * 16 + (lane >> 2) + 8 * h;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int n = n0 + 8 * j + 2 * qd;
            float val = v[h][2 * j], gate = v[h][2 * j + 1];
            if (g.bias != nullptr && n < g.N) { val += __ldg(g.bias + n); gate += __ldg(g.bias + n + 1); }
            const float o = gelu_erf(gate) * val;
            const float o1 = __shfl_xor_sync(0xffffffffu, o, 1);
            if ((qd & 1) == 0) {
              uint32_t hw, lw;
              if (g.u_scale > 0.f) split2u(o * g.u_scale, o1 * g.u_scale, hw, lw);
              else split2(o, o1, hw, lw);
              const int b = 8 * j + 2 * qd;         // byte of U column (8 j + 2 qd) / 2 in the row
              *reinterpret_cast<uint32_t*>(stage + r * 128 + ((((b >> 4) ^ (r & 7)) << 4) | (b & 15))) = hw;
            }
          }
        }
      }
      fence_async_smem();                       // this thread's stage writes -> visible to the TMA store
      wg_bar(bar);
      if (elected) store_planes<H1>(tmUh, tmUl, stage, n0 >> 1, m0 + half * 64, g.c_seg);
    }
  } else {
    // plain: (+bias)(+residual).  residual may alias C, so the compiler may not move a residual load above a store to C:
    // a load after a store waits out its own round trip to L2.  Every load of the half is therefore issued before its
    // first store; that stays correct in place because each element is read and written by the same thread.  The sums
    // go into v row by row, so a row's residual needs registers only until it is added (no spills in ping-pong, where
    // the other half's accumulators are live).
    const bool bias = g.bias != nullptr, res = g.residual != nullptr;
    float2 bb[BN / 8];
    long long prow[2];
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int n = n0 + 8 * j + 2 * qd;
      bb[j] = bias && n < g.N ? __ldg(reinterpret_cast<const float2*>(g.bias + n)) : make_float2(0.f, 0.f);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = mrow[h];
      prow[h] = map_row(m < g.M ? m : 0, g.c_seg, g.c_seg_stride, g.c_seg_off);
      float2 rr[BN / 8];
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int n = n0 + 8 * j + 2 * qd;
        rr[j] = res && m < g.M && n < g.N ? *reinterpret_cast<const float2*>(g.residual + prow[h] * g.ldr + n)
                                          : make_float2(0.f, 0.f);
      }
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        if (bias) { v[h][2 * j] += bb[j].x; v[h][2 * j + 1] += bb[j].y; }
        if (res) { v[h][2 * j] += rr[j].x; v[h][2 * j + 1] += rr[j].y; }
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (mrow[h] < g.M) {
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int n = n0 + 8 * j + 2 * qd;
          if (n < g.N) *reinterpret_cast<float2*>(g.c + prow[h] * g.ldc + n) = make_float2(v[h][2 * j], v[h][2 * j + 1]);
        }
      }
    }
  }
}

template <bool TF32, int NACC, int EPI, bool H1 = false>
__global__ void __launch_bounds__(THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmAl,
                  const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmA2l,
                  const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl,
                  const __grid_constant__ CUtensorMap tmUh, const __grid_constant__ CUtensorMap tmUl, const Args g) {
  constexpr int BK = TF32 ? 32 : 64;          // elements per 128-byte row
  constexpr bool PINGPONG = !TF32 && NACC == 1;
  constexpr int HALVES = PINGPONG ? 2 : 1;    // 64-row halves of a tile one consumer warpgroup computes
  constexpr int A_BYTES = BM * 128, W_BYTES = BN * 128;
  constexpr uint32_t TX_BYTES = H1 ? A_BYTES + W_BYTES : TF32 ? A_BYTES + 2 * W_BYTES : 2 * A_BYTES + 2 * W_BYTES;
  constexpr int NS = stages<H1>(), SB = stage_bytes<H1>();
  constexpr int W_OFF = H1 ? A_BYTES : 2 * A_BYTES;   // W_hi in a stage (W_lo follows it)
  static_assert(!H1 || (!TF32 && NACC == 1), "the single-product form is the single-accumulator f16 kernel");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  __shared__ __align__(8) uint64_t full[NS], empty[NS];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int num_kb = g.K / BK;
  const int num_n_blk = (g.N + BN - 1) / BN;
  const int num_tiles = g.num_m_blk * num_n_blk;

  if (tid == 0) {
    prefetch_map(&tmA); prefetch_map(&tmA2); prefetch_map(&tmWh);
    if (!H1) prefetch_map(&tmWl);
    if (!TF32 && !H1) { prefetch_map(&tmAl); prefetch_map(&tmA2l); }
    for (int s = 0; s < NS; ++s) {
      mbar_init(&full[s], 1);                   // the producer's expect_tx
      mbar_init(&empty[s], PINGPONG ? 1 : 2);   // the warpgroup that owns the tile / both consumer warpgroups
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_sync();

  // Producer and consumers walk the same (tile, k-block) sequence; the running k-block count `it` alone gives the stage
  // (it % NS) and the phase parity ((it / NS) & 1) of its full barrier.  The producer waits on the phase before
  // it: a fresh empty barrier counts as released.
  // n fastest: W (at most a few MB of planes) stays in L2 while the CTAs running at the same time share the rows of A,
  // so A is read from HBM about once.  (m fastest re-reads all of A per n block once A outgrows L2.)
  auto tile_origin = [&](int t, int& m0, int& n0) { m0 = (t / num_n_blk) * BM; n0 = (t % num_n_blk) * BN; };

  if (warp < 4) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (tid == 0) {
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int m0, n0;
        tile_origin(tile, m0, n0);
        const bool second = n0 >= g.n_split;    // dual-A: columns >= n_split read the second matrix
        int c1[2], c2[2];                       // TMA coordinates of the two 64-row boxes of A (row map)
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
          const int r = m0 + hf * 64;
          if (g.a_seg > 0) { c1[hf] = r % g.a_seg; c2[hf] = r / g.a_seg; }
          else { c1[hf] = r; c2[hf] = 0; }
        }
        const CUtensorMap* mah = second ? &tmA2 : &tmA;
        const CUtensorMap* mal = second ? &tmA2l : &tmAl;
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const int s = it % NS;
          uint8_t* sp = smem + (size_t)s * SB;
          mbar_wait(&empty[s], ((it / NS) & 1) ^ 1);
          mbar_expect_tx(&full[s], TX_BYTES);
          tma_load_3d(mah, &full[s], sp, kb * BK, c1[0], c2[0]);
          tma_load_3d(mah, &full[s], sp + A_BYTES / 2, kb * BK, c1[1], c2[1]);
          if (!TF32 && !H1) {
            tma_load_3d(mal, &full[s], sp + A_BYTES, kb * BK, c1[0], c2[0]);
            tma_load_3d(mal, &full[s], sp + A_BYTES + A_BYTES / 2, kb * BK, c1[1], c2[1]);
          }
          tma_load_2d(&tmWh, &full[s], sp + W_OFF, kb * BK, n0);
          if (!H1) tma_load_2d(&tmWl, &full[s], sp + W_OFF + W_BYTES, kb * BK, n0);
        }
      }
    }
  } else {
    setmaxnreg_inc<CONSUMER_REGS>();
    // consumer warpgroup: ping-pong, the tiles j = wg, wg + 2, ... of the CTA's walk; cooperative, rows [64 wg, +64) of
    // every tile
    const int wg = (warp >> 2) - 1;
    auto release = [&](uint32_t i) {            // the wgmmas of k-block i have retired: free its stage
      if ((tid & 127) == 0) mbar_arrive(&empty[i % NS]);
    };
    // Ping-pong order: before each tile but the CTA's first, a warpgroup waits on its barrier ORDER_BAR + wg; the owner
    // of the previous tile arrives on it once it has issued that tile's last k-block, and only if a next tile exists, so
    // every arrival meets exactly one wait.  The chain also keeps the consumers' full-barrier waits in k-block order.
    uint32_t it = PINGPONG ? wg * num_kb : 0;
    for (int tile = blockIdx.x + (PINGPONG ? wg : 0) * gridDim.x; tile < num_tiles; tile += (PINGPONG ? 2 : 1) * gridDim.x) {
      int m0, n0;
      tile_origin(tile, m0, n0);
      const bool second = n0 >= g.n_split;
      float acc[HALVES][BN / 2], crs[NACC == 2 ? BN / 2 : 1];
#pragma unroll
      for (int h = 0; h < HALVES; ++h)
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[h][i] = 0.f;
#pragma unroll
      for (int i = 0; i < (NACC == 2 ? BN / 2 : 1); ++i) crs[i] = 0.f;
      if (PINGPONG && tile != (int)blockIdx.x) named_bar_sync(ORDER_BAR + wg, 256);

      for (int kb = 0; kb < num_kb; ++kb, ++it) {
        const int s = it % NS;
        uint8_t* sp = smem + (size_t)s * SB;
        mbar_wait(&full[s], (it / NS) & 1);
        if (TF32) {
          // this warpgroup's 64 rows of A (one 8 KiB box): tf32 hi in place, lo into the A_lo slot
          float4* a = reinterpret_cast<float4*>(sp + wg * (A_BYTES / 2));
          float4* alo = reinterpret_cast<float4*>(sp + A_BYTES + wg * (A_BYTES / 2));
          const int t = tid & 127;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int idx = t + i * 128;
            const float4 v = a[idx];
            float4 hi, lo;
            hi.x = tf32_rn(v.x); hi.y = tf32_rn(v.y); hi.z = tf32_rn(v.z); hi.w = tf32_rn(v.w);
            lo.x = v.x - hi.x; lo.y = v.y - hi.y; lo.z = v.z - hi.z; lo.w = v.w - hi.w;
            a[idx] = hi;
            alo[idx] = lo;
          }
          fence_async_smem();
          wg_bar(1 + wg);
        }
        const uint32_t sa = smem_u32(sp);
        const uint64_t d_whi = desc_sw128(sa + W_OFF), d_wlo = desc_sw128(sa + W_OFF + W_BYTES);
        wg_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {             // 32 bytes of the 128-byte row per MMA
          const uint64_t adv = (uint64_t)(k * 2);
#pragma unroll
          for (int h = 0; h < HALVES; ++h) {      // rows [64 r, +64) of the tile
            const int r = PINGPONG ? h : wg;
            const uint64_t d_ahi = desc_sw128(sa + r * (A_BYTES / 2)), d_alo = desc_sw128(sa + A_BYTES + r * (A_BYTES / 2));
            if constexpr (H1) {
              wgmma_f16_n128(acc[h], d_ahi + adv, d_whi + adv, 1);
            } else if constexpr (TF32) {
              wgmma_tf32_n128(acc[h], d_alo + adv, d_whi + adv, 1);
              wgmma_tf32_n128(acc[h], d_ahi + adv, d_wlo + adv, 1);
              wgmma_tf32_n128(acc[h], d_ahi + adv, d_whi + adv, 1);
            } else if constexpr (NACC == 2) {
              wgmma_f16_n128(crs, d_alo + adv, d_whi + adv, 1);
              wgmma_f16_n128(crs, d_ahi + adv, d_wlo + adv, 1);
              wgmma_f16_n128(acc[h], d_ahi + adv, d_whi + adv, 1);
            } else {
              wgmma_f16_n128(acc[h], d_alo + adv, d_whi + adv, 1);
              wgmma_f16_n128(acc[h], d_ahi + adv, d_wlo + adv, 1);
              wgmma_f16_n128(acc[h], d_ahi + adv, d_whi + adv, 1);
            }
          }
        }
        wg_commit();
        wg_wait<1>();
        if (kb > 0) release(it - 1);
      }
      // every wgmma of the tile is issued: the other warpgroup may start the next tile while this one drains
      if (PINGPONG && tile + (int)gridDim.x < num_tiles) named_bar_arrive(ORDER_BAR + (wg ^ 1), 256);
      wg_wait<0>();
      release(it - 1);
      if (PINGPONG) it += num_kb;               // the k-blocks of the other warpgroup's tile
#pragma unroll
      for (int h = 0; h < HALVES; ++h)
        epilogue<TF32, NACC, EPI, H1>(g, acc[h], crs, m0, n0, second, PINGPONG ? h : wg, warp, lane,
                                      smem + NS * SB + wg * EPI_STAGE_BYTES, 1 + wg, &tmUh, &tmUl);
    }
    // the warpgroup's TMA stores must be done before its shared memory goes away with the CTA
    if (tma_planes<TF32, EPI, H1>() && (tid & 127) == 0) bulk_wait<0>();
  }
}

// [K, seg, n_seg] map over a row-mapped matrix of 16-bit (esize 2) or fp32 (esize 4) elements, 128-byte x box_rows boxes
static inline int row_map(CUtensorMap* m, CUtensorMapDataType dt, int esize, const void* ptr, int ld, int rows, int cols,
                          int seg, int seg_stride, int seg_off, int box_rows = 64) {
  const int s = seg > 0 ? seg : rows;
  const int nseg = seg > 0 ? rows / seg : 1;
  const long long sstride = seg > 0 ? seg_stride : rows;
  cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)s, (cuuint64_t)nseg};
  cuuint64_t strides[2] = {(cuuint64_t)ld * esize, (cuuint64_t)sstride * ld * esize};
  cuuint32_t box[3] = {(cuuint32_t)(128 / esize), (cuuint32_t)box_rows, 1};
  const uint8_t* base = static_cast<const uint8_t*>(ptr) + (size_t)(seg > 0 ? seg_off : 0) * ld * esize;
  return encode_tiled(m, dt, base, 3, dims, strides, box);
}

// W [n_pad, K] (rows padded to a multiple of 128), 128-byte x 128-row boxes
static inline int w_map(CUtensorMap* m, CUtensorMapDataType dt, int esize, const void* ptr, int n_pad, int K) {
  cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)n_pad};
  cuuint64_t strides[1] = {(cuuint64_t)K * esize};
  cuuint32_t box[2] = {(cuuint32_t)(128 / esize), (cuuint32_t)BN};
  return encode_tiled(m, dt, ptr, 2, dims, strides, box);
}

// maps: A, A_lo, A2, A2_lo, W_hi, W_lo, and for the plane-writing f16 epilogues the output planes hi, lo (row_map with
// 32-row boxes); the other epilogues take six maps
template <bool TF32, int NACC, int EPI, bool H1 = false>
static int launch(const CUtensorMap* maps, const Args& g, cudaStream_t st) {
  auto kern = gemm_wgmma_kernel<TF32, NACC, EPI, H1>;
  constexpr int SMEM = smem_bytes<TF32, EPI, H1>();
  static KernelSetup setup;
  int resident = 0;
  const int rc = setup.resident(kern, THREADS, SMEM, &resident);
  if (rc != OMT_OK) return rc;
  const int tiles = g.num_m_blk * ((g.N + BN - 1) / BN);
  const dim3 grid(tiles < resident ? tiles : resident);
  const CUtensorMap& uh = tma_planes<TF32, EPI, H1>() ? maps[6] : maps[0];
  const CUtensorMap& ul = tma_planes<TF32, EPI, H1>() ? maps[7] : maps[0];
  OMT_CUDA(launch_k(kern, grid, dim3(THREADS), SMEM, st, maps[0], maps[1], maps[2], maps[3], maps[4], maps[5], uh, ul, g));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

}  // namespace wgg
}  // namespace omt
