// Attention v5: spatial (full, non-causal) attention core on sm_90a wgmma (f16) with row-scaled fp16 operand planes.
//   O = softmax(scale * Q K^T) V  per (sequence, head), head dim 64, N % 128 == 0
//   (F.scaled_dot_product_attention at modules/attention.py:451).
//
// Operands come from the QKV GEMM epilogue (gemm_wgmma.cuh, OMT_EPI_QKV_PLANES) already in tensor-core form:
//   q, k : after rope + l2norm + per-dim scale every component is bounded by max|q_scale| / max|k_scale|, so ONE static
//          power of two per layer puts them in fp16 range: planes hi = fp16(x * 2^e), lo = fp16(x * 2^e - hi)
//   v    : unbounded, scaled per (row, head); the inverse scales live in vinv[head][row]
// so S = Q K^T and O_j = P_j V_j each take THREE f16 wgmmas per 16-deep k-step into ONE fp32 accumulator
// (lo.hi, hi.lo, hi.hi in that order).
//   * K and V tiles come straight from TMA; V is consumed as an MN-MAJOR B operand (the token-major [64 keys][64 dims]
//     tile the TMA lands is the canonical SWIZZLE_128B MN-major layout), so nothing is transposed anywhere.
//   * the per-key inverse V scale is folded into P: P'' = p * vinv_j * 2^ep with ONE power of two per (sequence, head)
//     taken from the largest vinv of the sequence, so p'' stays in fp16 range; 2^-ep comes off with the final 1 / row-sum.
//
// Envelope (tests/attn_f16_cases.py derives the bound, tests/test_gpu_attn_f16_edges.py checks it): a key whose vinv is
// 2^-r of its sequence's largest gets P'' = p 2^(14 - r), so its share falls toward fp16's subnormal floor of 2^-24
// as r grows.  Worst |O - O_fp64| over softmax(...) |v| of the output, measured on an H100 SXM (error) next to the
// derived bound (bound), on the spread cases:
//   vinv spread 2^2  (the model's layers: within 2^2, |logits| below 7):  x3 error 4.2e-7, bound 2.4e-5;
//                                                                          x1 error 1.1e-4, bound 7.9e-3
//   vinv spread 2^32 (v rows 2^30 apart):                                  x3 error 3.2e-3, bound 3.2e-2;
//                                                                          x1 error 3.6e-3, bound 6.2e-2
//
// Warp-specialised and persistent.  One CTA per SM walks the work items (128-query tile, head, sequence) with a static
// stride.  Warpgroup 0 is the producer: its first warp finds each item's largest vinv and issues every load (Q by TMA
// into one buffer, K / V by TMA and the tile's 64 vinv by a bulk copy into a STAGES-deep full / empty mbarrier ring),
// running ahead into the next item while the consumers finish the current one.  Warpgroups 1 and 2 each own 64 query
// rows of the item and run decoupled, with no CTA barrier in the key loop:
//   * Q hi / lo are copied from shared memory into registers once per item (the A fragments of every Q.K^T wgmma); the
//     Q buffer is handed back as soon as both warpgroups have them.
//   * S_{j+1} = Q K_{j+1}^T is issued before the softmax of S_j (two S register arrays), so the tensor pipe works while
//     the softmax runs.  P'' hi / lo are packed from the S accumulator straight into the A fragments of the P.V wgmmas.
//   * a K / V stage is released once the P.V wgmmas that read it have retired.
// Every output row sees the same products in the same order as a serial loop over the key tiles would give it.
//
// H1 = true (omt_attn_spatial_h1, "f16x1", the throughput mode): the same kernel on the hi planes alone.  S = Q_hi.K_hi^T
// and O += P''_hi.V_hi take ONE wgmma per k-step, the ring carries K_hi / V_hi and vinv only (twice the stages in less
// shared memory), and O leaves as fp32 or as a hi plane.  The per-(row, head) V scale and the P'' packing are unchanged:
// they keep P.V in fp16 range whatever the number of products.
#include "omt_common.cuh"
#include "tc_ptx.cuh"
#include <cuda.h>

namespace omt {
int g_attn_f16_ctas = 2;      // omt_set_option("attn_f16_ctas", 1 | 2): accepted for compatibility (one kernel shape on sm_90)
namespace af16 {
using namespace omt::ptx;

constexpr int QT = 128, KT = 64, D = 64;
constexpr int TILE = KT * D * 2;                    // 8 KiB: one 64 x 64 fp16 plane tile
constexpr int THREADS = 384;                        // warpgroup 0: producer; 1, 2: consumers
// Shared memory of the two forms; PL = planes per operand (hi / lo, or hi alone)
template <bool H1> struct Smem {
  static constexpr int PL = H1 ? 1 : 2;
  static constexpr int STAGES = H1 ? 8 : 4;
  static constexpr int STAGE = 2 * PL * TILE;                   // K planes | V planes of one key tile
  static constexpr int OFF_Q = 0;                               // Q_hi [2 warpgroups] | Q_lo [2]
  static constexpr int OFF_KV = 2 * PL * TILE;                  // [STAGES] x (K_hi | K_lo | V_hi | V_lo)
  static constexpr int OFF_VI = OFF_KV + STAGES * STAGE;        // [STAGES] x the 64 vinv of the tile's keys
  static constexpr int OFF_CTRL = OFF_VI + STAGES * KT * 4;     // mbarriers, the item's largest vinv
  static constexpr int SMEM = OFF_CTRL + (H1 ? 256 : 128) + 1024;   // + alignment slack
  static constexpr uint32_t Q_BYTES = 2 * PL * TILE;
  static constexpr uint32_t KV_BYTES = STAGE + KT * 4;
  static_assert((2 + 2 * STAGES) * 8 + 4 <= (H1 ? 256 : 128), "control block");
};
// __launch_bounds__(384, 1) caps the kernel at 168 registers a thread: 40 * 128 + 232 * 256 == 168 * 384
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;

struct Args {
  const float* vinv;                                       // [heads][rows] inverse scales of the v rows
  long long rows;                                          // n_seq * N
  float* o; uint16_t* o_hi; uint16_t* o_lo; int ldo;
  int N, heads, items;                                     // items = n_seq * heads * N / QT
  float scale_log2;                                        // scale * log2(e) / (q plane scale * k plane scale)
};

template <bool H1>
__global__ void __launch_bounds__(THREADS, 1)
attn_f16_kernel(const __grid_constant__ CUtensorMap tmQh, const __grid_constant__ CUtensorMap tmQl,
                const __grid_constant__ CUtensorMap tmKh, const __grid_constant__ CUtensorMap tmKl,
                const __grid_constant__ CUtensorMap tmVh, const __grid_constant__ CUtensorMap tmVl, const Args a) {
  using L = Smem<H1>;
  constexpr int PL = L::PL, STAGES = L::STAGES, OFF_Q = L::OFF_Q, OFF_KV = L::OFF_KV, OFF_VI = L::OFF_VI;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::OFF_CTRL);
  uint64_t& q_full = bars[0];                                         // Q planes (and vmax) of an item landed
  uint64_t& q_empty = bars[1];                                        // every consumer thread has its Q fragments
  uint64_t* full = bars + 2;                                          // [STAGES] K / V planes and vinv of a key tile landed
  uint64_t* empty = full + STAGES;                                    // [STAGES] both consumer warpgroups are done with it
  float* vmax = reinterpret_cast<float*>(bars + 2 + 2 * STAGES);      // largest vinv of the item's (sequence, head)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int ntiles = a.N / KT, nqt = a.N / QT;

  if (tid == 0) {
    if (H1) { prefetch_map(&tmQh); prefetch_map(&tmKh); prefetch_map(&tmVh); }
    else { prefetch_map(&tmQh); prefetch_map(&tmQl); prefetch_map(&tmKh); prefetch_map(&tmKl); prefetch_map(&tmVh); prefetch_map(&tmVl); }
    mbar_init(&q_full, 1);
    mbar_init(&q_empty, 256);
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_sync();

  // work item -> query tile (fastest), head, sequence: the CTAs running at once share a (sequence, head)'s K / V in L2
  auto decode = [&](int item, int& row_q0, int& row_k0, int& col0, int& head) {
    const int qt = item % nqt, hs = item / nqt, seq = hs / a.heads;
    head = hs % a.heads;
    row_k0 = seq * a.N;
    row_q0 = row_k0 + qt * QT;
    col0 = head * D;
  };

  // Producer and consumers walk the same items and key tiles; the running tile count `it` alone gives the stage
  // (it % STAGES) and the phase parity ((it / STAGES) & 1) of its full barrier, the item count `c` the parity of the Q
  // barriers.  The producer waits on the phase before it: a fresh empty barrier counts as released.
  if (warp < 4) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == 0) {
      uint32_t it = 0, c = 0;
      for (int item = blockIdx.x; item < a.items; item += gridDim.x, ++c) {
        int row_q0, row_k0, col0, head;
        decode(item, row_q0, row_k0, col0, head);
        const float* vinv_h = a.vinv + (size_t)head * a.rows + row_k0;
        float vmx = 0.f;
        for (int i = 4 * lane; i < a.N; i += 128) {
          const float4 v = __ldg(reinterpret_cast<const float4*>(vinv_h + i));
          vmx = fmaxf(vmx, fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)));
        }
        vmx = warp_max(vmx);
        mbar_wait(&q_empty, (c & 1) ^ 1);
        if (lane == 0) {
          *vmax = vmx;                                                // published by the arrive below
          mbar_expect_tx(&q_full, L::Q_BYTES);
          for (int w = 0; w < 2; ++w) {
            tma_load_2d(&tmQh, &q_full, smem + OFF_Q + w * TILE, col0, row_q0 + w * 64);
            if (!H1) tma_load_2d(&tmQl, &q_full, smem + OFF_Q + (2 + w) * TILE, col0, row_q0 + w * 64);
          }
        }
        for (int j = 0; j < ntiles; ++j, ++it) {
          const int s = it % STAGES;
          mbar_wait(&empty[s], ((it / STAGES) & 1) ^ 1);
          if (lane == 0) {
            uint8_t* sp = smem + OFF_KV + s * L::STAGE;
            const int kr = row_k0 + j * KT;
            mbar_expect_tx(&full[s], L::KV_BYTES);
            tma_load_2d(&tmKh, &full[s], sp, col0, kr);
            if (!H1) tma_load_2d(&tmKl, &full[s], sp + TILE, col0, kr);
            tma_load_2d(&tmVh, &full[s], sp + PL * TILE, col0, kr);
            if (!H1) tma_load_2d(&tmVl, &full[s], sp + 3 * TILE, col0, kr);
            bulk_load(smem + OFF_VI + s * KT * 4, vinv_h + j * KT, KT * 4, &full[s]);
          }
        }
      }
    }
  } else {
    setmaxnreg_inc<CONSUMER_REGS>();
    const int wg = (warp >> 2) - 1, qd = lane & 3;
    const int rl0 = (warp & 3) * 16 + (lane >> 2);   // this thread's rows (rl0, rl0 + 8) inside the warpgroup's 64
    const uint32_t sb = smem_u32(smem);
    auto release = [&](uint32_t t) {                 // the wgmmas that read running tile t have retired: free its stage
      if ((tid & 127) == 0) mbar_arrive(&empty[t % STAGES]);
    };
    // S of one key tile.  The first wgmma of a tile overwrites it, but it is defined once here: ptxas serialises the
    // wgmmas of a kernel whose accumulator registers can be undefined when a wgmma reads them.
    float sv[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) sv[i] = 0.f;
    uint32_t it = 0, c = 0;
    for (int item = blockIdx.x; item < a.items; item += gridDim.x, ++c) {
      int row_q0, row_k0, col0, head;
      decode(item, row_q0, row_k0, col0, head);
      mbar_wait(&q_full, c & 1);
      float p_scale, p_inv;
      row_scale(*vmax, p_scale, p_inv);              // p * vinv_j * p_scale <= 2^15 for every key (p <= 1)
      // Q A fragments, qh[4 kk + 2 e + h]: rows rl0 + 8 h, columns 16 kk + 8 e + 2 qd (+1), i.e. 16-byte chunk 2 kk + e
      // of the 128-byte row, stored at chunk (2 kk + e) ^ (row & 7) by the 128-byte swizzle
      uint32_t qh[16], ql[16];
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
#pragma unroll
        for (int e = 0; e < 2; ++e)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = rl0 + 8 * h;
            const uint8_t* p = smem + OFF_Q + wg * TILE + r * 128 + (((2 * kk + e) ^ (r & 7)) << 4) + qd * 4;
            qh[4 * kk + 2 * e + h] = *reinterpret_cast<const uint32_t*>(p);
            if (!H1) ql[4 * kk + 2 * e + h] = *reinterpret_cast<const uint32_t*>(p + 2 * TILE);
          }
      mbar_arrive(&q_empty);

      float o_acc[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) o_acc[i] = 0.f;
      float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
      uint32_t p_a[PL][16], p_b[PL][16];             // P'' hi (/ lo) A fragments of two tiles, laid out like qh / ql
      float alpha[2];

      auto wait_full = [&](uint32_t t) { mbar_wait(&full[t % STAGES], (t / STAGES) & 1); };
      auto issue_s = [&](uint32_t t) {               // S = Q . K^T of running tile t
        const uint32_t kv = sb + OFF_KV + (t % STAGES) * L::STAGE;
        const uint64_t dk_hi = desc_sw128(kv), dk_lo = desc_sw128(kv + TILE);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {             // 16 of the 64 head dims per MMA
          const uint64_t adv = (uint64_t)(kk * 2);
          if constexpr (H1) {
            wgmma_f16_n64_ra<0>(sv, qh + 4 * kk, dk_hi + adv, kk != 0);
          } else {
            wgmma_f16_n64_ra<0>(sv, ql + 4 * kk, dk_hi + adv, kk != 0);
            wgmma_f16_n64_ra<0>(sv, qh + 4 * kk, dk_lo + adv, 1);
            wgmma_f16_n64_ra<0>(sv, qh + 4 * kk, dk_hi + adv, 1);
          }
        }
      };
      auto issue_pv = [&](const uint32_t (&p)[PL][16], uint32_t t) {    // O += P''_t . V_t
        const uint32_t vh = sb + OFF_KV + (t % STAGES) * L::STAGE + PL * TILE, vl = vh + TILE;
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {             // 16 keys per MMA: 16 rows of the MN-major V tile = 2 KiB
          const uint64_t dvh = desc_sw128(vh + kk * 2048), dvl = desc_sw128(vl + kk * 2048);
          if constexpr (H1) {
            wgmma_f16_n64_ra<1>(o_acc, p[0] + 4 * kk, dvh, 1);
          } else {
            wgmma_f16_n64_ra<1>(o_acc, p[PL - 1] + 4 * kk, dvh, 1);
            wgmma_f16_n64_ra<1>(o_acc, p[0] + 4 * kk, dvl, 1);
            wgmma_f16_n64_ra<1>(o_acc, p[0] + 4 * kk, dvh, 1);
          }
        }
      };
      // online softmax of S (running tile t) into alpha, m_run, l_run and the P'' fragments p: a row's 64 keys sit in the
      // 4 lanes of a quad (16 each).  O *= alpha is left to the caller, once the P.V wgmmas of the tile before retired.
      auto softmax = [&](uint32_t (&p)[PL][16], uint32_t t) {
        float nm[2];
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
        const float* vi = reinterpret_cast<const float*>(smem + OFF_VI + (t % STAGES) * KT * 4);
        float ps[2] = {0.f, 0.f};
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const float2 w = *reinterpret_cast<const float2*>(vi + 8 * jj + 2 * qd);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const float e0 = ex2_fast((sv[4 * jj + 2 * h] + nm[h]) * a.scale_log2);      // the row maximum maps to exactly 1
            const float e1 = ex2_fast((sv[4 * jj + 2 * h + 1] + nm[h]) * a.scale_log2);
            ps[h] += e0 + e1;
            // keys 8 jj + 2 qd (+1) of row rl0 + 8 h: word 2 (jj & 1) + h of k-step jj / 2
            const int wd = 4 * (jj >> 1) + 2 * (jj & 1) + h;
            if constexpr (H1) p[0][wd] = pack_f16x2_sat(e0 * (w.x * p_scale), e1 * (w.y * p_scale));
            else split2u(e0 * (w.x * p_scale), e1 * (w.y * p_scale), p[0][wd], p[PL - 1][wd]);
          }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) l_run[h] = fmaf(l_run[h], alpha[h], ps[h]);     // partial row sum over this lane's keys
      };
      auto rescale = [&]() {
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) { o_acc[4 * jj + 2 * h] *= alpha[h]; o_acc[4 * jj + 2 * h + 1] *= alpha[h]; }
      };
      // tile j, its P'' in p: issue S_{j+1} (if `next`) and P''_j . V_j, run the softmax of S_{j+1} into pn while
      // P''_j . V_j is in flight, then retire both and free tile j's stage.  Nothing is in flight between two steps.
      auto step = [&](const uint32_t (&p)[PL][16], uint32_t (&pn)[PL][16], int j, bool next) {
        const uint32_t t = it + j;
        if (next) wait_full(t + 1);
        reg_fence(sv);
        reg_fence(o_acc);
        wg_fence();
        if (next) {
          issue_s(t + 1);
          wg_commit();
        }
        issue_pv(p, t);
        wg_commit();
        if (next) {
          wg_wait<1>();
          reg_fence(sv);
          softmax(pn, t + 1);
        }
        wg_wait<0>();
        reg_fence(o_acc);
        release(t);
        if (next) rescale();
      };

      wait_full(it);
      reg_fence(sv);
      wg_fence();
      issue_s(it);
      wg_commit();
      wg_wait<0>();
      reg_fence(sv);
      softmax(p_a, it);
      rescale();
      int j = 0;
      for (; j + 2 < ntiles; j += 2) {               // ntiles is even (N % 128 == 0)
        step(p_a, p_b, j, true);
        step(p_b, p_a, j + 1, true);
      }
      step(p_a, p_b, j, true);
      step(p_b, p_a, j + 1, false);
      it += ntiles;

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
          if (H1 && a.o_hi != nullptr) *reinterpret_cast<uint32_t*>(a.o_hi + ooff + 8 * jj) = pack_f16x2_sat(ov.x, ov.y);
          else if (a.o_hi != nullptr) store_split2(a.o_hi, a.o_lo, ooff + 8 * jj, ov);
          else *reinterpret_cast<float2*>(a.o + ooff + 8 * jj) = ov;
        }
      }
    }
  }
}

static int encode2d(CUtensorMap* m, const uint16_t* base, int cols, long long rows, int ld) {
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)KT};
  return encode_tiled(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, base, 2, dims, strides, box);
}

// Launch of either form: h1 takes the hi planes alone (the lo pointers are NULL and their maps never loaded).
template <bool H1>
static int launch(const char* who, const uint16_t* q_hi, const uint16_t* q_lo, int ldq, const uint16_t* k_hi,
                  const uint16_t* k_lo, int ldk, const uint16_t* v_hi, const uint16_t* v_lo, int ldv, const float* vinv,
                  float qk_plane_scale, float* o, uint16_t* o_hi, uint16_t* o_lo, int ldo, int n_seq, int N, int heads,
                  float scale, cudaStream_t stream) {
  using L = Smem<H1>;
  OMT_REQUIRE(N > 0 && N % QT == 0, "%s: N=%d must be a multiple of 128", who, N);
  OMT_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 4 == 0, "%s: bad leading dims", who);
  OMT_REQUIRE(((uintptr_t)q_hi | (uintptr_t)q_lo | (uintptr_t)k_hi | (uintptr_t)k_lo | (uintptr_t)v_hi | (uintptr_t)v_lo | (uintptr_t)vinv |
               (uintptr_t)o | (uintptr_t)o_hi | (uintptr_t)o_lo) % 16 == 0, "%s: pointers must be 16-byte aligned", who);
  OMT_REQUIRE(heads > 0 && heads <= 65535 && n_seq <= 65535 && qk_plane_scale > 0.f, "%s: bad arguments", who);
  if (n_seq == 0) return OMT_OK;
  const long long rows = (long long)n_seq * N;
  const long long items = rows / QT * heads;
  OMT_REQUIRE(rows < (1LL << 31) && items < (1LL << 31), "%s: n_seq * N = %lld rows is too many", who, rows);
  CUtensorMap tmQh, tmQl, tmKh, tmKl, tmVh, tmVl;
  int rc;
  if ((rc = encode2d(&tmQh, q_hi, heads * D, rows, ldq))) return rc;
  if ((rc = encode2d(&tmKh, k_hi, heads * D, rows, ldk))) return rc;
  if ((rc = encode2d(&tmVh, v_hi, heads * D, rows, ldv))) return rc;
  if (H1) {
    tmQl = tmQh; tmKl = tmKh; tmVl = tmVh;
  } else {
    if ((rc = encode2d(&tmQl, q_lo, heads * D, rows, ldq))) return rc;
    if ((rc = encode2d(&tmKl, k_lo, heads * D, rows, ldk))) return rc;
    if ((rc = encode2d(&tmVl, v_lo, heads * D, rows, ldv))) return rc;
  }
  static KernelSetup setup;
  int resident = 0;
  if ((rc = setup.resident(attn_f16_kernel<H1>, THREADS, L::SMEM, &resident))) return rc;
  Args a{vinv, rows, o, o_hi, o_lo, ldo, N, heads, (int)items, scale * 1.4426950408889634f / qk_plane_scale};
  const dim3 grid(items < resident ? (int)items : resident);
  OMT_CUDA(launch_k(attn_f16_kernel<H1>, grid, dim3(THREADS), L::SMEM, stream, tmQh, tmQl, tmKh, tmKl, tmVh, tmVl, a));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

}  // namespace af16
}  // namespace omt

using namespace omt;

extern "C" int omt_attn_spatial_h(const uint16_t* q_hi, const uint16_t* q_lo, int ldq, const uint16_t* k_hi,
                                  const uint16_t* k_lo, int ldk, const uint16_t* v_hi, const uint16_t* v_lo, int ldv,
                                  const float* vinv, float qk_plane_scale, float* o, uint16_t* o_hi, uint16_t* o_lo, int ldo,
                                  int n_seq, int N, int heads, float scale, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(q_hi && q_lo && k_hi && k_lo && v_hi && v_lo && vinv && (o || o_hi) && ((o_hi == nullptr) == (o_lo == nullptr)),
              "omt_attn_spatial_h: null pointer");
  return af16::launch<false>("omt_attn_spatial_h", q_hi, q_lo, ldq, k_hi, k_lo, ldk, v_hi, v_lo, ldv, vinv, qk_plane_scale,
                             o, o_hi, o_lo, ldo, n_seq, N, heads, scale, (cudaStream_t)stream);
}

extern "C" int omt_attn_spatial_h1(const uint16_t* q_hi, int ldq, const uint16_t* k_hi, int ldk, const uint16_t* v_hi,
                                   int ldv, const float* vinv, float qk_plane_scale, float* o, uint16_t* o_hi, int ldo,
                                   int n_seq, int N, int heads, float scale, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(q_hi && k_hi && v_hi && vinv && (o || o_hi), "omt_attn_spatial_h1: null pointer");
  return af16::launch<true>("omt_attn_spatial_h1", q_hi, nullptr, ldq, k_hi, nullptr, ldk, v_hi, nullptr, ldv, vinv,
                            qk_plane_scale, o, o_hi, nullptr, ldo, n_seq, N, heads, scale, (cudaStream_t)stream);
}

