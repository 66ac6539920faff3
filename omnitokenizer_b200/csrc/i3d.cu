// The I3D feature network of the FVD metric (OmniTokenizer/fvd/pytorch_i3d.py) on channels-last fp32 activations
// [B][T][H][W][Cs] (Cs: the channel count padded to a multiple of 32, or 4 for the 3-channel network input):
//
//   omt_conv3d     Unit3D (conv3d with TF-style SAME padding, BatchNorm folded into W and a bias, ReLU): an implicit GEMM
//                  C[M = B To Ho Wo, Cout] = A[M, K] . W[Cout, K]^T with K ordered (dt, dh, dw, c), in 3xTF32 on wgmma.
//   omt_maxpool3d  MaxPool3dSamePadding (F.pad with zeros, then max_pool3d), exact.
//   omt_i3d_head   AvgPool3d([2, 7, 7], stride 1) -> the `logits` 1x1x1 conv with bias -> mean over time.
//
// omt_conv3d is the warp-specialised persistent kernel of gemm_wgmma.cuh with its A producer replaced: instead of one
// thread issuing TMA boxes, the 128 producer threads each own one row of the 128-row tile (one output voxel) and gather
// its 128-byte k-block straight from the activation with 16-byte cp.async, zero-filled outside the volume (the
// reference's SAME padding is zero padding, pad // 2 in front and the rest behind, pytorch_i3d.py:93-124).  The bytes
// land in the 128B-swizzled K-major layout a TMA box would give; each thread then arrives on the stage's full barrier
// when its copies complete (cp.async.mbarrier.arrive.noinc).  W (BN-folded, pre-split into tf32 hi / lo) still comes by
// TMA.  The consumers are the cooperative 3xTF32 consumers: each warpgroup splits its 64 rows of A into tf32 hi / lo in
// shared memory and issues A_lo.W_hi + A_hi.W_lo + A_hi.W_hi per k-step, and every PROMOTE k-blocks adds the wgmma
// accumulator into a CUDA-core fp32 sum (see PROMOTE).  Cout <= 64 layers run a 64-wide N tile.
#include "gemm_wgmma.cuh"

namespace omt {
namespace i3d {
using namespace omt::ptx;

constexpr int BM = 128, THREADS = 384, STAGES = 3;
constexpr int A_BYTES = BM * 128;
template <int BN> __host__ __device__ constexpr int stage_bytes() { return 2 * A_BYTES + 2 * BN * 128; }   // A, A_lo, W_hi, W_lo
template <int BN> __host__ __device__ constexpr int smem_bytes() { return STAGES * stage_bytes<BN>() + 1024; }
// the gather producer needs more than a TMA issuer: 56 * 128 + 216 * 256 <= 168 * 384
constexpr int PRODUCER_REGS = 56, CONSUMER_REGS = 216;
// The tensor core's fp32 accumulation does not round to nearest: over a whole K (up to 3 x 5184 products a column) its
// error grows with K and reached 8e-4 of the I3D logits.  The accumulator is therefore restarted every PROMOTE k-blocks
// (24 wgmmas) and the chunk sums are added in fp32 on the CUDA cores, rounded to nearest.
constexpr int PROMOTE = 2;

struct ConvArgs {
  const float* x; int Cs;                       // input [B][T][H][W][Cs]
  int T, H, W;
  int To, Ho, Wo;
  int kt, kh, kw, st, sh, sw, pt, ph, pw;       // kernel, stride, front padding
  int M, N, K, taps;
  const float* bias;
  float* c; int ldc;                            // output row m, column n at c[m * ldc + n], n < N only
  int relu;
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool full) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(full ? 16 : 0) : "memory");
}
// arrives on `bar` once every cp.async this thread issued before has landed; counts as one of the barrier's arrivals
__device__ __forceinline__ void cp_async_arrive(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}

template <int BN>
__global__ void __launch_bounds__(THREADS, 1)
conv3d_kernel(const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl, const ConvArgs g) {
  constexpr int SB = stage_bytes<BN>(), W_BYTES = BN * 128;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  __shared__ __align__(8) uint64_t full[STAGES], empty[STAGES];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int num_kb = g.K / 32;
  const int num_n_blk = (g.N + BN - 1) / BN;
  const int num_tiles = ((g.M + BM - 1) / BM) * num_n_blk;

  if (tid == 0) {
    prefetch_map(&tmWh); prefetch_map(&tmWl);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 128 + 1);             // 128 gathering threads + the W expect_tx
      mbar_init(&empty[s], 2);                  // both consumer warpgroups
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_sync();

  if (warp < 4) {
    setmaxnreg_dec<PRODUCER_REGS>();
    const int t = tid;                          // this thread's row of every tile
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m0 = (tile / num_n_blk) * BM, n0 = (tile % num_n_blk) * BN;
      const int m = m0 + t;
      const bool row_ok = m < g.M;
      int r = row_ok ? m : 0;
      const int wo = r % g.Wo; r /= g.Wo;
      const int ho = r % g.Ho; r /= g.Ho;
      const int to = r % g.To, b = r / g.To;
      const int t0 = to * g.st - g.pt, h0 = ho * g.sh - g.ph, w0 = wo * g.sw - g.pw;
      const float* xb = g.x + (size_t)b * g.T * g.H * g.W * g.Cs;
      for (int kb = 0; kb < num_kb; ++kb, ++it) {
        const int s = it % STAGES;
        uint8_t* sp = smem + (size_t)s * SB;
        mbar_wait(&empty[s], ((it / STAGES) & 1) ^ 1);
        if (t == 0) {
          mbar_expect_tx(&full[s], 2 * W_BYTES);
          tma_load_2d(&tmWh, &full[s], sp + 2 * A_BYTES, kb * 32, n0);
          tma_load_2d(&tmWl, &full[s], sp + 2 * A_BYTES + W_BYTES, kb * 32, n0);
        }
        // row t at t * 128 bytes, its 16-byte chunk j at chunk j ^ (t & 7): the SWIZZLE_128B layout of a TMA box
        const uint32_t row = smem_u32(sp) + t * 128;
        if (g.Cs >= 32) {                       // one tap, 32 consecutive channels
          const int cpb = g.Cs >> 5;
          const int tap = kb / cpb, cb = kb - tap * cpb;
          const int dw = tap % g.kw, q = tap / g.kw;
          const int dh = q % g.kh, dt = q / g.kh;
          const int ti = t0 + dt, hi = h0 + dh, wi = w0 + dw;
          const bool in = row_ok && (unsigned)ti < (unsigned)g.T && (unsigned)hi < (unsigned)g.H && (unsigned)wi < (unsigned)g.W;
          const float* src = in ? xb + (((size_t)ti * g.H + hi) * g.W + wi) * g.Cs + cb * 32 : g.x;
#pragma unroll
          for (int j = 0; j < 8; ++j) cp_async16(row + ((j ^ (t & 7)) << 4), in ? src + 4 * j : g.x, in);
        } else {                                // Cs == 4: eight taps of one 16-byte granule each
#pragma unroll 1
          for (int j = 0; j < 8; ++j) {
            const int tap = kb * 8 + j;
            const int dw = tap % g.kw, q = tap / g.kw;
            const int dh = q % g.kh, dt = q / g.kh;
            const int ti = t0 + dt, hi = h0 + dh, wi = w0 + dw;
            const bool in = row_ok && tap < g.taps && (unsigned)ti < (unsigned)g.T && (unsigned)hi < (unsigned)g.H &&
                            (unsigned)wi < (unsigned)g.W;
            const float* src = in ? xb + (((size_t)ti * g.H + hi) * g.W + wi) * 4 : g.x;
            cp_async16(row + ((j ^ (t & 7)) << 4), src, in);
          }
        }
        cp_async_arrive(&full[s]);
      }
    }
  } else {
    setmaxnreg_inc<CONSUMER_REGS>();
    const int wg = (warp >> 2) - 1;             // rows [64 wg, +64) of every tile
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m0 = (tile / num_n_blk) * BM, n0 = (tile % num_n_blk) * BN;
      // acc: the tensor core's sum over one chunk of PROMOTE k-blocks; tot: the chunk sums, added on the CUDA cores
      float acc[BN / 2], tot[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) tot[i] = acc[i] = 0.f;
      bool pending = false;                     // the previous k-block's stage is not released yet
      for (int kb = 0; kb < num_kb; ++kb, ++it) {
        const int s = it % STAGES;
        uint8_t* sp = smem + (size_t)s * SB;
        mbar_wait(&full[s], (it / STAGES) & 1);
        {
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
        const uint64_t d_whi = desc_sw128(sa + 2 * A_BYTES), d_wlo = desc_sw128(sa + 2 * A_BYTES + W_BYTES);
        const uint64_t d_ahi = desc_sw128(sa + wg * (A_BYTES / 2)), d_alo = desc_sw128(sa + A_BYTES + wg * (A_BYTES / 2));
        const uint32_t chunk_d = (kb % PROMOTE) != 0;   // 0: the chunk's first k-step overwrites acc
        wg_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint64_t adv = (uint64_t)(k * 2);
          if constexpr (BN == 128) {
            wgmma_tf32_n128(acc, d_alo + adv, d_whi + adv, k == 0 ? chunk_d : 1u);
            wgmma_tf32_n128(acc, d_ahi + adv, d_wlo + adv, 1);
            wgmma_tf32_n128(acc, d_ahi + adv, d_whi + adv, 1);
          } else {
            wgmma_tf32_n64(acc, d_alo + adv, d_whi + adv, k == 0 ? chunk_d : 1u);
            wgmma_tf32_n64(acc, d_ahi + adv, d_wlo + adv, 1);
            wgmma_tf32_n64(acc, d_ahi + adv, d_whi + adv, 1);
          }
        }
        wg_commit();
        if ((kb + 1) % PROMOTE == 0 || kb + 1 == num_kb) {
          wg_wait<0>();
          reg_fence(acc);
          if ((tid & 127) == 0) {
            if (pending) mbar_arrive(&empty[(it - 1) % STAGES]);
            mbar_arrive(&empty[it % STAGES]);
          }
          pending = false;
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) tot[i] += acc[i];
        } else {
          wg_wait<1>();
          if (pending && (tid & 127) == 0) mbar_arrive(&empty[(it - 1) % STAGES]);
          pending = true;
        }
      }
      // bias (+ ReLU); columns n < N only: the next branch's slice of a concat buffer starts at N
      const int qd = lane & 3;
      const int mr = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = mr + 8 * h;
        if (m >= g.M) continue;
        float* crow = g.c + (size_t)m * g.ldc;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int n = n0 + 8 * j + 2 * qd;
          if (n < g.N) {
            const float2 bb = __ldg(reinterpret_cast<const float2*>(g.bias + n));
            float v0 = tot[4 * j + 2 * h] + bb.x, v1 = tot[4 * j + 2 * h + 1] + bb.y;
            if (g.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
            *reinterpret_cast<float2*>(crow + n) = make_float2(v0, v1);
          }
        }
      }
    }
  }
}

template <int BN>
int launch_conv(const ConvArgs& g, const float* w_hi, const float* w_lo, cudaStream_t st) {
  auto kern = conv3d_kernel<BN>;
  constexpr int SMEM = smem_bytes<BN>();
  static int resident[64];
  int dev = 0;
  OMT_CUDA(cudaGetDevice(&dev));
  OMT_REQUIRE(dev >= 0 && dev < 64, "omt_conv3d: device ordinal %d out of range", dev);
  if (resident[dev] == 0) {
    OMT_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    int per_sm = 0, sms = 0;
    OMT_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, THREADS, SMEM));
    OMT_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    OMT_REQUIRE(per_sm > 0, "omt_conv3d: no CTA fits on an SM of device %d", dev);
    resident[dev] = per_sm * sms;
  }
  const int n_pad = (g.N + 127) / 128 * 128;
  CUtensorMap maps[2];
  cuuint64_t dims[2] = {(cuuint64_t)g.K, (cuuint64_t)n_pad};
  cuuint64_t strides[1] = {(cuuint64_t)g.K * 4};
  cuuint32_t box[2] = {32, (cuuint32_t)BN};
  int rc;
  if ((rc = wgg::encode_map(&maps[0], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, w_hi, 2, dims, strides, box))) return rc;
  if ((rc = wgg::encode_map(&maps[1], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, w_lo, 2, dims, strides, box))) return rc;
  const int tiles = ((g.M + BM - 1) / BM) * ((g.N + BN - 1) / BN);
  const dim3 grid(tiles < resident[dev] ? tiles : resident[dev]);
  OMT_CUDA(launch_k(kern, grid, dim3(THREADS), SMEM, st, maps[0], maps[1], g));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

// MaxPool3dSamePadding on channels-last fp32: one thread per 4 channels of an output voxel.  Taps outside the volume
// read F.pad's zeros; max_pool3d's CPU rule (maxval from -inf, replaced when val > maxval or val is NaN) in (t, h, w)
// order, so ties and signed zeros resolve as torch resolves them.
__global__ void __launch_bounds__(256)
maxpool3d_kernel(const float4* __restrict__ x, float4* __restrict__ y, int C4, long long total, int T, int H, int W,
                 int To, int Ho, int Wo, int kt, int kh, int kw, int st, int sh, int sw, int pt, int ph, int pw) {
  pdl_sync();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4);
    long long r = i / C4;
    const int wo = (int)(r % Wo); r /= Wo;
    const int ho = (int)(r % Ho); r /= Ho;
    const int to = (int)(r % To);
    const long long b = r / To;
    float m[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
    for (int dt = 0; dt < kt; ++dt) {
      const int ti = to * st - pt + dt;
      for (int dh = 0; dh < kh; ++dh) {
        const int hi = ho * sh - ph + dh;
        for (int dw = 0; dw < kw; ++dw) {
          const int wi = wo * sw - pw + dw;
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if ((unsigned)ti < (unsigned)T && (unsigned)hi < (unsigned)H && (unsigned)wi < (unsigned)W)
            v = __ldg(x + (((b * T + ti) * H + hi) * W + wi) * C4 + c);
          const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (e[k] > m[k] || isnan(e[k])) m[k] = e[k];
        }
      }
    }
    y[i] = make_float4(m[0], m[1], m[2], m[3]);
  }
}

// AvgPool3d([2, 7, 7], stride 1) over x [B][T][7][7][Cs] (sum in (t, h, w) order, then / 98), the logits conv
// W[N][C] . p + bias per time step, then the mean over the T - 1 steps.  One CTA per clip; a warp per class.
constexpr int HEAD_THREADS = 256;
__global__ void __launch_bounds__(HEAD_THREADS)
i3d_head_kernel(const float* __restrict__ x, int Cs, int C, int T, const float* __restrict__ w,
                const float* __restrict__ bias, int N, float* __restrict__ out) {
  extern __shared__ float sh[];
  float* pooled = sh;           // [C]
  float* acc = sh + C;          // [N]
  pdl_sync();
  const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int n = tid; n < N; n += HEAD_THREADS) acc[n] = 0.f;
  const float* xb = x + (size_t)b * T * 49 * Cs;
  for (int t = 0; t + 1 < T; ++t) {
    __syncthreads();
    for (int c = tid; c < C; c += HEAD_THREADS) {
      float s = 0.f;
      for (int dt = 0; dt < 2; ++dt)
        for (int p = 0; p < 49; ++p) s += __ldg(xb + ((size_t)(t + dt) * 49 + p) * Cs + c);
      pooled[c] = s / 98.f;
    }
    __syncthreads();
    for (int n = warp; n < N; n += HEAD_THREADS / 32) {
      const float* wn = w + (size_t)n * C;
      float s = 0.f;
      for (int c = lane; c < C; c += 32) s = fmaf(__ldg(wn + c), pooled[c], s);
      s = warp_sum(s);
      if (lane == 0) acc[n] += s + __ldg(bias + n);
    }
  }
  __syncthreads();
  for (int n = tid; n < N; n += HEAD_THREADS) out[(size_t)b * N + n] = acc[n] / (float)(T - 1);
}

// 2-D pooling of the FID InceptionV3 (pytorch-fid inception.py) on channels-last fp32 [B][H][W][Cs]: one thread per 4
// channels of an output pixel.  Only taps inside the image take part (max: padding never wins; average: the count
// excludes it, count_include_pad=False), in (h, w) order as torch's CPU kernels visit them: max_pool2d's rule (maxval
// from -inf, replaced when val > maxval or val is NaN); avg_pool2d's fp32 sum from 0, then one true division by the count.
// Output pixel p, channel c at y[p * ldy + c]: a pool branch writes its slice of the concat buffer in place.
__global__ void __launch_bounds__(256)
pool2d_kernel(const float4* __restrict__ x, float* __restrict__ y, int Cs4, int C4, int ldy, long long total, int H,
              int W, int Ho, int Wo, int kh, int kw, int sh, int sw, int ph, int pw, int avg) {
  pdl_sync();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4);
    const long long p = i / C4;                   // output pixel (b, ho, wo)
    const int wo = (int)(p % Wo);
    const long long r = p / Wo;
    const int ho = (int)(r % Ho);
    const long long b = r / Ho;
    const int h0 = ho * sh - ph, w0 = wo * sw - pw;
    const int hs = max(h0, 0), he = min(h0 + kh, H), ws = max(w0, 0), we = min(w0 + kw, W);
    const float init = avg ? 0.f : -INFINITY;
    float m[4] = {init, init, init, init};
    for (int hi = hs; hi < he; ++hi) {
      for (int wi = ws; wi < we; ++wi) {
        const float4 v = __ldg(x + ((b * H + hi) * W + wi) * Cs4 + c);
        const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          if (avg) m[k] = __fadd_rn(m[k], e[k]);
          else if (e[k] > m[k] || isnan(e[k])) m[k] = e[k];
        }
      }
    }
    if (avg) {
      const float n = (float)((he - hs) * (we - ws));
#pragma unroll
      for (int k = 0; k < 4; ++k) m[k] = __fdiv_rn(m[k], n);
    }
    *reinterpret_cast<float4*>(y + p * ldy + 4 * c) = make_float4(m[0], m[1], m[2], m[3]);
  }
}

}  // namespace i3d
}  // namespace omt

using namespace omt;

extern "C" int omt_conv3d(const float* x, int Cs, int B, int T, int H, int W, const float* w_hi, const float* w_lo,
                          int K, const float* bias, int N, int kt, int kh, int kw, int st, int sh, int sw, int pt,
                          int ph, int pw, int To, int Ho, int Wo, float* y, int ldy, int relu, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(x && w_hi && w_lo && bias && y, "omt_conv3d: null pointer");
  OMT_REQUIRE(Cs == 4 || (Cs >= 32 && Cs % 32 == 0), "omt_conv3d: input channel stride %d must be 4 or a multiple of 32", Cs);
  OMT_REQUIRE(B >= 1 && T >= 1 && H >= 1 && W >= 1 && To >= 1 && Ho >= 1 && Wo >= 1,
              "omt_conv3d: input %dx%dx%dx%d, output %dx%dx%d", B, T, H, W, To, Ho, Wo);
  OMT_REQUIRE(kt >= 1 && kh >= 1 && kw >= 1 && st >= 1 && sh >= 1 && sw >= 1 && pt >= 0 && ph >= 0 && pw >= 0 &&
                  pt < kt && ph < kh && pw < kw,
              "omt_conv3d: kernel %dx%dx%d, stride %dx%dx%d, front padding %dx%dx%d", kt, kh, kw, st, sh, sw, pt, ph, pw);
  OMT_REQUIRE((long long)(To - 1) * st - pt < T && (long long)(Ho - 1) * sh - ph < H && (long long)(Wo - 1) * sw - pw < W,
              "omt_conv3d: output %dx%dx%d reads past the %dx%dx%d input", To, Ho, Wo, T, H, W);
  const int taps = kt * kh * kw;
  const long long k_need = Cs == 4 ? ((long long)taps * 4 + 31) / 32 * 32 : (long long)taps * Cs;
  OMT_REQUIRE(K == k_need, "omt_conv3d: K=%d, expected %lld for %d taps of %d channels", K, k_need, taps, Cs);
  const long long M = (long long)B * To * Ho * Wo;
  OMT_REQUIRE(M <= 0x7fffffffLL && (long long)B * T * H * W * Cs <= 0x7fffffffffffLL, "omt_conv3d: %lld output rows", M);
  OMT_REQUIRE(N >= 2 && N % 2 == 0 && ldy >= N && ldy % 2 == 0, "omt_conv3d: N=%d must be even and <= ldy=%d (even)", N, ldy);
  OMT_REQUIRE(aligned_to(16, {x, w_hi, w_lo}) && aligned_to(8, {bias, y}),
              "omt_conv3d: x / w_hi / w_lo must be 16-byte and bias / y 8-byte aligned");
  i3d::ConvArgs g{};
  g.x = x; g.Cs = Cs; g.T = T; g.H = H; g.W = W; g.To = To; g.Ho = Ho; g.Wo = Wo;
  g.kt = kt; g.kh = kh; g.kw = kw; g.st = st; g.sh = sh; g.sw = sw; g.pt = pt; g.ph = ph; g.pw = pw;
  g.M = (int)M; g.N = N; g.K = K; g.taps = taps;
  g.bias = bias; g.c = y; g.ldc = ldy; g.relu = relu ? 1 : 0;
  if (N <= 64) return i3d::launch_conv<64>(g, w_hi, w_lo, (cudaStream_t)stream);
  return i3d::launch_conv<128>(g, w_hi, w_lo, (cudaStream_t)stream);
}

extern "C" int omt_maxpool3d(const float* x, int Cs, int B, int T, int H, int W, int kt, int kh, int kw, int st, int sh,
                             int sw, int pt, int ph, int pw, int To, int Ho, int Wo, float* y, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(x && y, "omt_maxpool3d: null pointer");
  OMT_REQUIRE(Cs >= 4 && Cs % 4 == 0, "omt_maxpool3d: channel stride %d must be a multiple of 4", Cs);
  OMT_REQUIRE(B >= 1 && T >= 1 && H >= 1 && W >= 1 && To >= 1 && Ho >= 1 && Wo >= 1,
              "omt_maxpool3d: input %dx%dx%dx%d, output %dx%dx%d", B, T, H, W, To, Ho, Wo);
  OMT_REQUIRE(kt >= 1 && kh >= 1 && kw >= 1 && st >= 1 && sh >= 1 && sw >= 1 && pt >= 0 && ph >= 0 && pw >= 0,
              "omt_maxpool3d: window %dx%dx%d, stride %dx%dx%d, front padding %dx%dx%d", kt, kh, kw, st, sh, sw, pt, ph, pw);
  OMT_REQUIRE(aligned_to(16, {x, y}), "omt_maxpool3d: x and y must be 16-byte aligned");
  const long long total = (long long)B * To * Ho * Wo * (Cs / 4);
  const long long blocks = (total + 255) / 256;
  const int grid = (int)(blocks < 65536 ? blocks : 65536);
  OMT_CUDA(launch_k(i3d::maxpool3d_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)stream,
                    reinterpret_cast<const float4*>(x), reinterpret_cast<float4*>(y), Cs / 4, total, T, H, W, To, Ho, Wo,
                    kt, kh, kw, st, sh, sw, pt, ph, pw));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

extern "C" int omt_i3d_head(const float* x, int Cs, int C, int B, int T, const float* w, const float* bias, int N,
                            float* out, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(x && w && bias && out, "omt_i3d_head: null pointer");
  OMT_REQUIRE(B >= 1 && B <= 65535 && T >= 2 && C >= 1 && Cs >= C && N >= 1,
              "omt_i3d_head: B=%d, T=%d (>= 2: the average pool spans 2 frames), C=%d of stride %d, N=%d", B, T, C, Cs, N);
  const size_t smem = (size_t)(C + N) * sizeof(float);
  OMT_REQUIRE(smem <= 48 * 1024, "omt_i3d_head: C=%d + N=%d floats exceed 48 KiB of shared memory", C, N);
  OMT_CUDA(launch_k(i3d::i3d_head_kernel, dim3(B), dim3(i3d::HEAD_THREADS), smem, (cudaStream_t)stream, x, Cs, C, T, w,
                    bias, N, out));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

extern "C" int omt_pool2d(const float* x, int Cs, int C, int B, int H, int W, int kh, int kw, int sh, int sw, int ph,
                          int pw, int Ho, int Wo, float* y, int ldy, int mode, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(x && y, "omt_pool2d: null pointer");
  OMT_REQUIRE(mode == OMT_POOL_MAX || mode == OMT_POOL_AVG, "omt_pool2d: mode %d is neither max (0) nor average (1)", mode);
  OMT_REQUIRE(Cs % 4 == 0 && C >= 4 && C % 4 == 0 && C <= Cs && ldy >= C && ldy % 4 == 0,
              "omt_pool2d: C=%d channels of stride %d into rows of %d: all multiples of 4, C <= both", C, Cs, ldy);
  OMT_REQUIRE(B >= 1 && H >= 1 && W >= 1 && Ho >= 1 && Wo >= 1, "omt_pool2d: input %dx%dx%d, output %dx%d", B, H, W, Ho, Wo);
  OMT_REQUIRE(kh >= 1 && kw >= 1 && sh >= 1 && sw >= 1 && ph >= 0 && pw >= 0 && 2 * ph <= kh && 2 * pw <= kw,
              "omt_pool2d: window %dx%d, stride %dx%d, padding %dx%d (at most half the window)", kh, kw, sh, sw, ph, pw);
  OMT_REQUIRE((long long)(Ho - 1) * sh - ph + kh <= H + 2LL * ph && (long long)(Wo - 1) * sw - pw + kw <= W + 2LL * pw,
              "omt_pool2d: output %dx%d reads past the %dx%d input padded by %dx%d", Ho, Wo, H, W, ph, pw);
  OMT_REQUIRE(aligned_to(16, {x, y}), "omt_pool2d: x and y (at its column offset) must be 16-byte aligned");
  const long long total = (long long)B * Ho * Wo * (C / 4);
  const long long blocks = (total + 255) / 256;
  const int grid = (int)(blocks < 65536 ? blocks : 65536);
  OMT_CUDA(launch_k(i3d::pool2d_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)stream, reinterpret_cast<const float4*>(x),
                    y, Cs / 4, C / 4, ldy, total, H, W, Ho, Wo, kh, kw, sh, sw, ph, pw, mode == OMT_POOL_AVG ? 1 : 0));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}
