// Per-frame reconstruction metrics of evaluation/common_metrics_on_video_quality (PSNR, SSIM) and the tokenizer's own
// LPIPS (OmniTokenizer/modules/lpips.py, VGG16 + five 1x1 "lin" layers) on frame pairs (P, H, W, 3), channels last.
//
//   omt_psnr_ssim    one CTA per frame pair: the fp64 sum of squared differences over the whole frame, and the mean of
//                    calculate_ssim.py's SSIM map per channel over the valid (H - 10) x (W - 10) crop, built from five
//                    11-tap Gaussian-filtered maps (separable, fp64).  Tiles of 32 x 32 outputs: the (42 x 42) fp32
//                    input halo of both images, then the five horizontally filtered rows [42][32] in fp64.
//   omt_lpips_input  calculate_lpips.py's x * 2 - 1 and ScalingLayer's (x - shift) / scale, fp32 in the reference's
//                    op order, into the [P][H][W][4] network input of omt_conv3d (channel 3 zero).
//   omt_lpips_head   normalize_tensor of both images' features at one VGG tap, the squared difference, NetLinLayer's
//                    1x1 conv and spatial_average: one CTA per pair, a warp per pixel.
//   omt_lpips_map    the same per-pixel term written as a map (the lpips package's spatial=True AlexNet LPIPS).
//   omt_lpips_upsample_mean  the five tap maps upsampled to the frame (torch's bilinear, align_corners=False), summed
//                    in tap order, and each pair's mean over the frame in fp64: one CTA per pair.
//   omt_softmax_rows  the Inception Score classifier's softmax: one CTA per row.
//   omt_inception_score  the IS split reduction in fp64: the split's column means (a thread per column), then one CTA
//                    per split, a warp per row, for the rows' KL divergences from the split's marginal.
//
// Every reduction has a fixed order (per-thread partials in a fixed visiting order, then a fixed tree over the block):
// no floating-point atomics, so two runs give the same bits.
#include "omt_common.cuh"

namespace omt {
namespace quality {

constexpr int SS_TH = 32, SS_TW = 32, SS_R = 5, SS_TAPS = 2 * SS_R + 1;
constexpr int SS_IH = SS_TH + 2 * SS_R, SS_IW = SS_TW + 2 * SS_R;
constexpr int SS_THREADS = 256;
// the two images' input halo in fp32 (their values are fp32), the five horizontally filtered maps in fp64
constexpr int SS_SMEM = 2 * SS_IH * SS_IW * (int)sizeof(float) + 5 * SS_IH * SS_TW * (int)sizeof(double);

// value of element i (pixel * 3 + channel) of frame p: the fp32 value itself, or the byte looked up in the frame's table
template <bool F32>
__device__ __forceinline__ float load_value(const void* x, long long i, const float* lut_s) {
  if constexpr (F32) return __ldg(reinterpret_cast<const float*>(x) + i);
  else return lut_s[__ldg(reinterpret_cast<const uint8_t*>(x) + i)];
}

// fixed-order sum of v over the block into red[0] (every thread must call; returns the sum in every thread)
__device__ __forceinline__ double block_sum(double v, double* red) {
  const int tid = threadIdx.x;
  red[tid] = v;
  __syncthreads();
#pragma unroll
  for (int s = SS_THREADS / 2; s > 0; s >>= 1) {
    if (tid < s) red[tid] = __dadd_rn(red[tid], red[tid + s]);
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();
  return r;
}

// Fixed-order warp sum in fp64: the same butterfly in every lane, so every lane holds the same bits.
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

template <bool F32>
__global__ void __launch_bounds__(SS_THREADS, 2)
psnr_ssim_kernel(const void* __restrict__ a, const float* __restrict__ lut_a, const int32_t* __restrict__ sel_a,
                 const void* __restrict__ b, const float* __restrict__ lut_b, const int32_t* __restrict__ sel_b, int H,
                 int W, const double* __restrict__ taps, double* __restrict__ sse_out, double* __restrict__ ssim_out) {
  extern __shared__ __align__(16) uint8_t smem[];
  double* hs = reinterpret_cast<double*>(smem);                              // [5][SS_IH][SS_TW]
  float* ta = reinterpret_cast<float*>(hs + 5 * SS_IH * SS_TW);              // [SS_IH][SS_IW]
  float* tb = ta + SS_IH * SS_IW;
  __shared__ float la[256], lb[256];
  __shared__ double k[SS_TAPS];
  __shared__ double red[SS_THREADS];
  pdl_sync();
  const int p = blockIdx.x, tid = threadIdx.x;
  if (tid < SS_TAPS) k[tid] = taps[tid];
  if constexpr (!F32) {
    la[tid] = lut_a[(sel_a ? sel_a[p] : 0) * 256 + tid];
    lb[tid] = lut_b[(sel_b ? sel_b[p] : 0) * 256 + tid];
  }
  __syncthreads();
  const long long frame = (long long)H * W * 3;
  const void* fa = F32 ? (const void*)(reinterpret_cast<const float*>(a) + p * frame)
                       : (const void*)(reinterpret_cast<const uint8_t*>(a) + p * frame);
  const void* fb = F32 ? (const void*)(reinterpret_cast<const float*>(b) + p * frame)
                       : (const void*)(reinterpret_cast<const uint8_t*>(b) + p * frame);

  // img_psnr: the squared differences of the fp32 values, widened to fp64, over C H W
  double sse = 0.0;
  for (long long i = tid; i < frame; i += SS_THREADS) {
    const double d = (double)load_value<F32>(fa, i, la) - (double)load_value<F32>(fb, i, lb);
    sse = fma(d, d, sse);
  }
  sse = block_sum(sse, red);

  // ssim(): per channel, the mean of the SSIM map over the valid crop
  constexpr double C1 = 0.01 * 0.01, C2 = 0.03 * 0.03;
  const int Ho = H - 2 * SS_R, Wo = W - 2 * SS_R;
  const int tiles_x = (Wo + SS_TW - 1) / SS_TW, tiles = ((Ho + SS_TH - 1) / SS_TH) * tiles_x;
  double ch_sum = 0.0;                          // the channel means added in channel order: np.array(ssims).mean()
  for (int c = 0; c < 3; ++c) {
    double acc = 0.0;
    for (int t = 0; t < tiles; ++t) {
      const int y0 = (t / tiles_x) * SS_TH, x0 = (t % tiles_x) * SS_TW;
      for (int i = tid; i < SS_IH * SS_IW; i += SS_THREADS) {
        const int r = i / SS_IW, q = i - r * SS_IW;
        const int gy = y0 + r, gx = x0 + q;
        const bool in = gy < H && gx < W;
        const long long e = ((long long)gy * W + gx) * 3 + c;
        ta[i] = in ? load_value<F32>(fa, e, la) : 0.f;
        tb[i] = in ? load_value<F32>(fb, e, lb) : 0.f;
      }
      __syncthreads();
      // horizontal pass: every halo row, the tile's output columns
      for (int i = tid; i < SS_IH * SS_TW; i += SS_THREADS) {
        const int r = i / SS_TW, q = i - r * SS_TW;
        double m1 = 0.0, m2 = 0.0, e11 = 0.0, e22 = 0.0, e12 = 0.0;
#pragma unroll
        for (int j = 0; j < SS_TAPS; ++j) {
          const double x = (double)ta[r * SS_IW + q + j], y = (double)tb[r * SS_IW + q + j];
          const double kj = k[j];
          m1 = fma(kj, x, m1);
          m2 = fma(kj, y, m2);
          e11 = fma(kj, x * x, e11);             // x * x, y * y, x * y of fp32 values are exact in fp64
          e22 = fma(kj, y * y, e22);
          e12 = fma(kj, x * y, e12);
        }
        hs[(0 * SS_IH + r) * SS_TW + q] = m1;
        hs[(1 * SS_IH + r) * SS_TW + q] = m2;
        hs[(2 * SS_IH + r) * SS_TW + q] = e11;
        hs[(3 * SS_IH + r) * SS_TW + q] = e22;
        hs[(4 * SS_IH + r) * SS_TW + q] = e12;
      }
      __syncthreads();
      // vertical pass and the SSIM map (calculate_ssim.py:6-22 in its op order)
      for (int i = tid; i < SS_TH * SS_TW; i += SS_THREADS) {
        const int r = i / SS_TW, q = i - r * SS_TW;
        if (y0 + r >= Ho || x0 + q >= Wo) continue;
        double f[5];
#pragma unroll
        for (int m = 0; m < 5; ++m) {
          double s = 0.0;
#pragma unroll
          for (int j = 0; j < SS_TAPS; ++j) s = fma(k[j], hs[(m * SS_IH + r + j) * SS_TW + q], s);
          f[m] = s;
        }
        const double mu1_sq = __dmul_rn(f[0], f[0]), mu2_sq = __dmul_rn(f[1], f[1]), mu1_mu2 = __dmul_rn(f[0], f[1]);
        const double s1 = __dsub_rn(f[2], mu1_sq), s2 = __dsub_rn(f[3], mu2_sq), s12 = __dsub_rn(f[4], mu1_mu2);
        const double num = __dmul_rn(__dadd_rn(__dmul_rn(2.0, mu1_mu2), C1), __dadd_rn(__dmul_rn(2.0, s12), C2));
        const double den = __dmul_rn(__dadd_rn(__dadd_rn(mu1_sq, mu2_sq), C1), __dadd_rn(__dadd_rn(s1, s2), C2));
        acc = __dadd_rn(acc, __ddiv_rn(num, den));
      }
      __syncthreads();
    }
    ch_sum = __dadd_rn(ch_sum, block_sum(acc, red) / ((double)Ho * Wo));
  }
  if (tid == 0) {
    sse_out[p] = sse;
    ssim_out[p] = ch_sum / 3.0;
  }
}

// x * 2 - 1 (calculate_lpips.trans), then ScalingLayer's (x - shift_c) / scale_c, fp32 rounded after every op.  The u8
// form looks the whole chain up in a per-channel table built on the host with the same torch expression.
template <bool F32>
__global__ void __launch_bounds__(256)
lpips_input_kernel(const void* __restrict__ x, const float* __restrict__ lut, const int32_t* __restrict__ sel,
                   const float* __restrict__ shift_scale, long long pixels, long long frame_pixels,
                   float4* __restrict__ out) {
  pdl_sync();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < pixels; i += (long long)gridDim.x * blockDim.x) {
    float v[3];
    if constexpr (F32) {
      const float* xp = reinterpret_cast<const float*>(x) + i * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float t = __fsub_rn(__fmul_rn(__ldg(xp + c), 2.f), 1.f);
        v[c] = __fdiv_rn(__fsub_rn(t, __ldg(shift_scale + c)), __ldg(shift_scale + 3 + c));
      }
    } else {
      const uint8_t* xp = reinterpret_cast<const uint8_t*>(x) + i * 3;
      const float* l = lut + (sel ? (long long)sel[i / frame_pixels] : 0LL) * (3 * 256);
#pragma unroll
      for (int c = 0; c < 3; ++c) v[c] = __ldg(l + c * 256 + __ldg(xp + c));
    }
    out[i] = make_float4(v[0], v[1], v[2], 0.f);
  }
}

// One LPIPS pixel of a warp, features pa and pb of C channels:
//   sum_c w_c (x_c / (|x| + 1e-10) - y_c / (|y| + 1e-10))^2,  |x| = sqrt(sum_c x_c^2)   (fp32, true divisions)
// lane partials in channel order, then the warp butterfly: every lane returns the same bits.
__device__ __forceinline__ float lpips_pixel(const float* pa, const float* pb, int C, const float* __restrict__ lin_w,
                                             int lane) {
  float na = 0.f, nb = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float u = __ldg(pa + c), v = __ldg(pb + c);
    na = __fmaf_rn(u, u, na);
    nb = __fmaf_rn(v, v, nb);
  }
  const float da = __fadd_rn(__fsqrt_rn(warp_sum(na)), 1e-10f), db = __fadd_rn(__fsqrt_rn(warp_sum(nb)), 1e-10f);
  float s = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float d = __fsub_rn(__fdiv_rn(__ldg(pa + c), da), __fdiv_rn(__ldg(pb + c), db));
    s = __fmaf_rn(__ldg(lin_w + c), __fmul_rn(d, d), s);
  }
  return warp_sum(s);
}

// One VGG tap of P pairs, images i and i + P of x [2P][h][w][Cs]: lpips_pixel summed over the pixels in fp64 (warp
// partials in pixel order, then the warps in order) and divided by h w.
constexpr int HEAD_THREADS = 512, HEAD_WARPS = HEAD_THREADS / 32;
__global__ void __launch_bounds__(HEAD_THREADS)
lpips_head_kernel(const float* __restrict__ x, int Cs, int C, int P, int hw, const float* __restrict__ lin_w, int tap,
                  float* __restrict__ taps_out, float* __restrict__ total) {
  __shared__ double red[HEAD_WARPS];
  pdl_sync();
  const int p = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const float* xa = x + (size_t)p * hw * Cs;
  const float* xb = x + (size_t)(p + P) * hw * Cs;
  double acc = 0.0;
  for (int pix = warp; pix < hw; pix += HEAD_WARPS) {
    const float s = lpips_pixel(xa + (size_t)pix * Cs, xb + (size_t)pix * Cs, C, lin_w, lane);
    acc = __dadd_rn(acc, (double)s);
  }
  if (lane == 0) red[warp] = acc;
  __syncthreads();
  if (tid == 0) {
    double t = 0.0;
    for (int i = 0; i < HEAD_WARPS; ++i) t = __dadd_rn(t, red[i]);
    const float r = (float)(t / (double)hw);
    taps_out[(size_t)tap * P + p] = r;
    if (total) {                              // lpips.py:105-108: val = res[0]; val += res[1] ... in fp32
      float v = tap == 0 ? r : taps_out[p];
      for (int i = 1; i <= tap; ++i) v = __fadd_rn(v, i == tap ? r : taps_out[(size_t)i * P + p]);
      total[p] = v;
    }
  }
}

// The per-pixel map of one tap: a warp per pixel of the P h w, lane 0 stores lpips_pixel.
constexpr int MAP_THREADS = 256, MAP_WARPS = MAP_THREADS / 32;
__global__ void __launch_bounds__(MAP_THREADS)
lpips_map_kernel(const float* __restrict__ x, int Cs, int C, int P, int hw, const float* __restrict__ lin_w,
                 float* __restrict__ map) {
  pdl_sync();
  const int lane = threadIdx.x & 31;
  const long long n = (long long)P * hw;
  for (long long i = blockIdx.x * (long long)MAP_WARPS + (threadIdx.x >> 5); i < n; i += (long long)gridDim.x * MAP_WARPS) {
    const long long p = i / hw, pix = i - p * hw;
    const float s = lpips_pixel(x + (size_t)(p * hw + pix) * Cs, x + (size_t)((p + P) * hw + pix) * Cs, C, lin_w, lane);
    if (lane == 0) map[i] = s;
  }
}

// The spatial=True tail: one CTA per pair; thread t takes pixels t, t + UP_THREADS, ... in order, v = 0 + up_0 + ...
// + up_{n-1} (torch's upsample_bilinear2d_out_frame<float, float> per tap), and the fp64 sum of v over the frame is
// the per-thread partials, the warp butterfly, then the warps in order.
constexpr int UP_THREADS = 512, UP_WARPS = UP_THREADS / 32;
struct UpTaps {
  omt_lpips_tap t[OMT_LPIPS_MAX_TAPS];
  float sh[OMT_LPIPS_MAX_TAPS], sw[OMT_LPIPS_MAX_TAPS];   // (float)h / (float)H, (float)w / (float)W, as torch's host
};

// area_pixel_compute_source_index(scale, dst, align_corners=false, cubic=false) and its two taps and weights
__device__ __forceinline__ void bilinear_axis(float scale, int dst, int in, int& i0, int& i1, float& l0, float& l1) {
  float src = __fmaf_rn((float)dst + 0.5f, scale, -0.5f);
  src = src >= 0.f ? src : 0.f;
  i0 = (int)src;
  i1 = i0 + (i0 < in - 1 ? 1 : 0);
  l1 = __fsub_rn(src, (float)i0);
  l0 = __fsub_rn(1.f, l1);
}

__global__ void __launch_bounds__(UP_THREADS)
lpips_upsample_mean_kernel(UpTaps taps, int n_taps, int H, int W, float* __restrict__ map_out,
                           float* __restrict__ mean_out) {
  __shared__ double red[UP_WARPS];
  pdl_sync();
  const int p = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int hw = H * W;
  double acc = 0.0;
  for (int i = tid; i < hw; i += UP_THREADS) {
    const int y = i / W, x = i - y * W;
    float v = 0.f;
#pragma unroll
    for (int k = 0; k < OMT_LPIPS_MAX_TAPS; ++k) {
      if (k >= n_taps) break;
      const int h = taps.t[k].h, w = taps.t[k].w;
      const float* a = taps.t[k].map + (size_t)p * h * w;
      float up;
      if (h == H && w == W) {
        up = __ldg(a + i);
      } else {
        int y0, y1, x0, x1;
        float h0, h1, w0, w1;
        bilinear_axis(taps.sh[k], y, h, y0, y1, h0, h1);
        bilinear_axis(taps.sw[k], x, w, x0, x1, w0, w1);
        const float top = __fmaf_rn(w0, __ldg(a + y0 * w + x0), __fmul_rn(w1, __ldg(a + y0 * w + x1)));
        const float bot = __fmaf_rn(w0, __ldg(a + y1 * w + x0), __fmul_rn(w1, __ldg(a + y1 * w + x1)));
        up = __fmaf_rn(h0, top, __fmul_rn(h1, bot));
      }
      v = __fadd_rn(v, up);
    }
    if (map_out) map_out[(size_t)p * hw + i] = v;
    acc = __dadd_rn(acc, (double)v);
  }
  acc = warp_sum_d(acc);
  if (lane == 0) red[warp] = acc;
  __syncthreads();
  if (tid == 0) {
    double t = red[0];
    for (int i = 1; i < UP_WARPS; ++i) t = __dadd_rn(t, red[i]);
    mean_out[p] = (float)(t / (double)hw);
  }
}

// Row r of x -> row r of y: m = max, e = exp(x - m) in fp64 rounded to fp32 (a probability's error then does not grow
// with its distance from the max), the fp32 sum of e (per-thread partials in column order, the warp butterfly, then the
// warps in order), one true division per entry.
constexpr int SM_THREADS = 256, SM_WARPS = SM_THREADS / 32;
__global__ void __launch_bounds__(SM_THREADS, 1)
softmax_rows_kernel(const float* __restrict__ x, int ldx, int N, float* __restrict__ y, int ldy) {
  __shared__ float red[SM_WARPS];
  pdl_sync();
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const float* xr = x + (size_t)blockIdx.x * ldx;
  float* yr = y + (size_t)blockIdx.x * ldy;
  float m = -INFINITY;
  for (int j = tid; j < N; j += SM_THREADS) m = fmaxf(m, __ldg(xr + j));
  m = warp_max(m);
  if (lane == 0) red[warp] = m;
  __syncthreads();
  m = red[0];
#pragma unroll
  for (int i = 1; i < SM_WARPS; ++i) m = fmaxf(m, red[i]);
  __syncthreads();
  float s = 0.f;
  for (int j = tid; j < N; j += SM_THREADS) {
    const float e = (float)exp(__dsub_rn((double)__ldg(xr + j), (double)m));
    yr[j] = e;
    s = __fadd_rn(s, e);
  }
  s = warp_sum(s);
  if (lane == 0) red[warp] = s;
  __syncthreads();
  s = red[0];
#pragma unroll
  for (int i = 1; i < SM_WARPS; ++i) s = __fadd_rn(s, red[i]);
  for (int j = tid; j < N; j += SM_THREADS) yr[j] = __fdiv_rn(yr[j], s);
}

// py[k][j]: the fp64 sum of column j over split k's rows in row order, over n.
__global__ void __launch_bounds__(256)
is_col_mean_kernel(const float* __restrict__ p, int ldp, int N, int n, double* __restrict__ col_mean) {
  pdl_sync();
  const int k = blockIdx.y, j = blockIdx.x * 256 + threadIdx.x;
  if (j >= N) return;
  const float* pk = p + (size_t)k * n * ldp + j;
  double s = 0.0;
  for (int r = 0; r < n; ++r) s = __dadd_rn(s, (double)__ldg(pk + (size_t)r * ldp));
  col_mean[(size_t)k * N + j] = __ddiv_rn(s, (double)n);
}

// One CTA per split: y = py / sum(py) in shared memory, then warp w takes rows w, w + KL_WARPS, ... in order; a row's
// sum and its KL terms are lane partials in column order and the warp butterfly.  The warps' totals are added in order.
constexpr int KL_THREADS = 512, KL_WARPS = KL_THREADS / 32;
__global__ void __launch_bounds__(KL_THREADS)
is_kl_kernel(const float* __restrict__ p, int ldp, int N, int n, const double* __restrict__ col_mean,
             double* __restrict__ kl) {
  extern __shared__ double q[];                 // [N]
  __shared__ double red[KL_WARPS];
  pdl_sync();
  const int k = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const double* py = col_mean + (size_t)k * N;
  double s = 0.0;
  for (int j = tid; j < N; j += KL_THREADS) s = __dadd_rn(s, py[j]);
  s = warp_sum_d(s);
  if (lane == 0) red[warp] = s;
  __syncthreads();
  double tot = red[0];
  for (int i = 1; i < KL_WARPS; ++i) tot = __dadd_rn(tot, red[i]);
  for (int j = tid; j < N; j += KL_THREADS) q[j] = __ddiv_rn(py[j], tot);
  __syncthreads();
  double acc = 0.0;
  for (int r = warp; r < n; r += KL_WARPS) {
    const float* row = p + ((size_t)k * n + r) * ldp;
    double rs = 0.0;
    for (int j = lane; j < N; j += 32) rs = __dadd_rn(rs, (double)__ldg(row + j));
    rs = warp_sum_d(rs);
    double t = 0.0;
    for (int j = lane; j < N; j += 32) {
      const double xj = __ddiv_rn((double)__ldg(row + j), rs);
      // rel_entr: 0 where x == 0; where x > 0 the split's column mean, so y, is positive too
      if (xj > 0.0) t = __dadd_rn(t, __dmul_rn(xj, log(__ddiv_rn(xj, q[j]))));
    }
    acc = __dadd_rn(acc, warp_sum_d(t));
  }
  if (lane == 0) red[warp] = acc;
  __syncthreads();
  if (tid == 0) {
    double t = red[0];
    for (int i = 1; i < KL_WARPS; ++i) t = __dadd_rn(t, red[i]);
    kl[k] = __ddiv_rn(t, (double)n);
  }
}

}  // namespace quality
}  // namespace omt

using namespace omt;

extern "C" int omt_psnr_ssim(const void* a, const float* lut_a, const int32_t* sel_a, const void* b, const float* lut_b,
                             const int32_t* sel_b, int form, int P, int H, int W, const double* taps, double* sse,
                             double* ssim, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(a && b && taps && sse && ssim, "omt_psnr_ssim: null pointer");
  OMT_REQUIRE(form == OMT_Q_U8 || form == OMT_Q_F32, "omt_psnr_ssim: form %d is neither u8 (0) nor f32 (1)", form);
  OMT_REQUIRE(form == OMT_Q_F32 || (lut_a && lut_b), "omt_psnr_ssim: the u8 form needs both value tables");
  OMT_REQUIRE(form == OMT_Q_U8 || (!lut_a && !lut_b && !sel_a && !sel_b), "omt_psnr_ssim: the f32 form takes no tables");
  OMT_REQUIRE(P >= 1 && P <= 0x7fffffff && H >= quality::SS_TAPS && W >= quality::SS_TAPS,
              "omt_psnr_ssim: P=%d pairs of %dx%d (SSIM needs H, W >= 11)", P, H, W);
  OMT_REQUIRE((long long)H * W * 3 <= 0x7fffffffLL, "omt_psnr_ssim: %dx%d frames are too large", H, W);
  OMT_REQUIRE(aligned_to(form == OMT_Q_F32 ? 4 : 1, {a, b}) && aligned_to(4, {lut_a, lut_b, sel_a, sel_b}) &&
                  aligned_to(8, {taps, sse, ssim}),
              "omt_psnr_ssim: misaligned pointer");
  cudaStream_t st = (cudaStream_t)stream;
  static KernelSetup setup_u8, setup_f32;
  int rc;
  if ((rc = setup_u8.smem(quality::psnr_ssim_kernel<false>, quality::SS_SMEM))) return rc;
  if ((rc = setup_f32.smem(quality::psnr_ssim_kernel<true>, quality::SS_SMEM))) return rc;
  if (form == OMT_Q_F32)
    OMT_CUDA(launch_k(quality::psnr_ssim_kernel<true>, dim3(P), dim3(quality::SS_THREADS), quality::SS_SMEM, st, a, lut_a,
                      sel_a, b, lut_b, sel_b, H, W, taps, sse, ssim));
  else
    OMT_CUDA(launch_k(quality::psnr_ssim_kernel<false>, dim3(P), dim3(quality::SS_THREADS), quality::SS_SMEM, st, a, lut_a,
                      sel_a, b, lut_b, sel_b, H, W, taps, sse, ssim));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

extern "C" int omt_lpips_input(const void* x, const float* lut, const int32_t* sel, const float* shift_scale, int form,
                               int P, int H, int W, float* out, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(x && out, "omt_lpips_input: null pointer");
  OMT_REQUIRE(form == OMT_Q_U8 || form == OMT_Q_F32, "omt_lpips_input: form %d is neither u8 (0) nor f32 (1)", form);
  OMT_REQUIRE(form == OMT_Q_U8 ? (lut && !shift_scale) : (shift_scale && !lut && !sel),
              "omt_lpips_input: the u8 form takes lut (and sel), the f32 form shift_scale");
  OMT_REQUIRE(P >= 1 && H >= 1 && W >= 1, "omt_lpips_input: P=%d, %dx%d", P, H, W);
  OMT_REQUIRE(aligned_to(16, {out}) && aligned_to(4, {lut, sel, shift_scale}) && aligned_to(form == OMT_Q_F32 ? 4 : 1, {x}),
              "omt_lpips_input: out must be 16-byte aligned, x / tables 4-byte");
  const long long frame = (long long)H * W, pixels = frame * P;
  const long long blocks = (pixels + 255) / 256;
  const int grid = (int)(blocks < 65536 ? blocks : 65536);
  cudaStream_t st = (cudaStream_t)stream;
  if (form == OMT_Q_F32)
    OMT_CUDA(launch_k(quality::lpips_input_kernel<true>, dim3(grid), dim3(256), 0, st, x, lut, sel, shift_scale, pixels,
                      frame, reinterpret_cast<float4*>(out)));
  else
    OMT_CUDA(launch_k(quality::lpips_input_kernel<false>, dim3(grid), dim3(256), 0, st, x, lut, sel, shift_scale, pixels,
                      frame, reinterpret_cast<float4*>(out)));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

extern "C" int omt_lpips_head(const float* x, int Cs, int C, int P, int h, int w, const float* lin_w, int tap,
                              float* taps_out, float* total, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(x && lin_w && taps_out, "omt_lpips_head: null pointer");
  OMT_REQUIRE(C >= 1 && Cs >= C && P >= 1 && P <= 0x7fffffff && h >= 1 && w >= 1 && tap >= 0 && tap < 5,
              "omt_lpips_head: C=%d of stride %d, P=%d, %dx%d, tap %d", C, Cs, P, h, w, tap);
  OMT_REQUIRE((long long)h * w <= 0x7fffffffLL, "omt_lpips_head: %dx%d maps are too large", h, w);
  OMT_REQUIRE(aligned_to(4, {x, lin_w, taps_out, total}), "omt_lpips_head: misaligned pointer");
  OMT_CUDA(launch_k(quality::lpips_head_kernel, dim3(P), dim3(quality::HEAD_THREADS), 0, (cudaStream_t)stream, x, Cs, C, P,
                    h * w, lin_w, tap, taps_out, total));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

extern "C" int omt_lpips_map(const float* x, int Cs, int C, int P, int h, int w, const float* lin_w, float* map,
                             omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(x && lin_w && map, "omt_lpips_map: null pointer");
  OMT_REQUIRE(C >= 1 && Cs >= C && P >= 1 && h >= 1 && w >= 1, "omt_lpips_map: C=%d of stride %d, P=%d, %dx%d", C, Cs,
              P, h, w);
  OMT_REQUIRE((long long)h * w <= 0x7fffffffLL, "omt_lpips_map: %dx%d maps are too large", h, w);
  OMT_REQUIRE(aligned_to(4, {x, lin_w, map}), "omt_lpips_map: misaligned pointer");
  const long long warps = (long long)P * h * w;
  const long long blocks = (warps + quality::MAP_WARPS - 1) / quality::MAP_WARPS;
  const int grid = (int)(blocks < sm_count() * 16LL ? blocks : sm_count() * 16LL);
  OMT_CUDA(launch_k(quality::lpips_map_kernel, dim3(grid), dim3(quality::MAP_THREADS), 0, (cudaStream_t)stream, x, Cs, C,
                    P, h * w, lin_w, map));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

extern "C" int omt_lpips_upsample_mean(const omt_lpips_tap* taps, int n_taps, int P, int H, int W, float* map_out,
                                       float* mean_out, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(taps && mean_out, "omt_lpips_upsample_mean: null pointer");
  OMT_REQUIRE(n_taps >= 1 && n_taps <= OMT_LPIPS_MAX_TAPS, "omt_lpips_upsample_mean: %d taps (1 to %d)", n_taps,
              OMT_LPIPS_MAX_TAPS);
  OMT_REQUIRE(P >= 1 && H >= 1 && W >= 1 && (long long)H * W <= 0x7fffffffLL, "omt_lpips_upsample_mean: P=%d, %dx%d",
              P, H, W);
  OMT_REQUIRE(aligned_to(4, {map_out, mean_out}), "omt_lpips_upsample_mean: misaligned pointer");
  quality::UpTaps t{};
  for (int k = 0; k < n_taps; ++k) {
    const omt_lpips_tap& a = taps[k];
    OMT_REQUIRE(a.map, "omt_lpips_upsample_mean: tap %d: null map", k);
    OMT_REQUIRE(a.h >= 1 && a.w >= 1 && (long long)a.h * a.w <= 0x7fffffffLL, "omt_lpips_upsample_mean: tap %d is %dx%d",
                k, a.h, a.w);
    OMT_REQUIRE(aligned_to(4, {a.map}), "omt_lpips_upsample_mean: tap %d: misaligned map", k);
    t.t[k] = a;
    t.sh[k] = (float)a.h / (float)H;            // area_pixel_compute_scale<float>, align_corners=False, no scale given
    t.sw[k] = (float)a.w / (float)W;
  }
  OMT_CUDA(launch_k(quality::lpips_upsample_mean_kernel, dim3(P), dim3(quality::UP_THREADS), 0, (cudaStream_t)stream, t,
                    n_taps, H, W, map_out, mean_out));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

extern "C" int omt_softmax_rows(const float* x, int ldx, int rows, int N, float* y, int ldy, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(x && y, "omt_softmax_rows: null pointer");
  OMT_REQUIRE(rows >= 1 && N >= 1 && ldx >= N && ldy >= N, "omt_softmax_rows: %d rows of %d, ldx=%d, ldy=%d", rows, N,
              ldx, ldy);
  OMT_REQUIRE(aligned_to(4, {x, y}), "omt_softmax_rows: x and y must be 4-byte aligned");
  OMT_CUDA(launch_k(quality::softmax_rows_kernel, dim3(rows), dim3(quality::SM_THREADS), 0, (cudaStream_t)stream, x, ldx,
                    N, y, ldy));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

extern "C" int omt_inception_score(const float* p, int ldp, int N, int n, int splits, double* col_mean, double* kl,
                                   omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(p && col_mean && kl, "omt_inception_score: null pointer");
  OMT_REQUIRE(N >= 1 && ldp >= N && n >= 1 && splits >= 1 && splits <= 65535,
              "omt_inception_score: %d splits of %d rows of %d, ldp=%d", splits, n, N, ldp);
  const size_t smem = (size_t)N * sizeof(double);
  OMT_REQUIRE(smem <= 48 * 1024, "omt_inception_score: N=%d classes exceed 48 KiB of fp64 shared memory", N);
  OMT_REQUIRE(aligned_to(4, {p}) && aligned_to(8, {col_mean, kl}), "omt_inception_score: misaligned pointer");
  // the KL kernel's static red[] comes on top of q[N]: past N = 6128 the two exceed the 48 KiB a launch gets unasked
  static KernelSetup setup_kl;
  int rc;
  if ((rc = setup_kl.smem(quality::is_kl_kernel, 48 * 1024))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  OMT_CUDA(launch_k(quality::is_col_mean_kernel, dim3((N + 255) / 256, splits), dim3(256), 0, st, p, ldp, N, n,
                    col_mean));
  OMT_LAUNCH_CHECK();
  OMT_CUDA(launch_k(quality::is_kl_kernel, dim3(splits), dim3(quality::KL_THREADS), smem, st, p, ldp, N, n,
                    (const double*)col_mean, kl));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}
