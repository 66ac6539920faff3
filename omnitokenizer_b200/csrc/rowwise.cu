// Row-wise / HBM-bound kernels of the OmniTokenizer encode/decode path:
// LayerNorm, patch gather+LN, un-patchify, PEG gather-stencil, rope+l2norm+scale.
// All of them stream the canonical X[B][T'][N][C] buffer once with 16-byte accesses.
#include "omt_common.cuh"

namespace omt {

int g_peg_kernel = 4;   // omt_set_option("peg_kernel", 3|4): 4 = peg_tile4_kernel (cp.async gather + FFMA2, default), 3 = peg_tile_kernel

// ------------------------------------------------------------------------------------------
// Whole rows in a warp's registers, shared by LayerNorm and both patch gathers.
// ------------------------------------------------------------------------------------------
// Column of float4 chunk i of a lane's row.  PAIR (C a multiple of 256, NV = C / 128: 2, 4, 6 or 8): a lane owns 8
// consecutive columns per 256-column block (two adjacent float4 chunks), so the row-scaled planes leave as 16-byte stores
// (512 B per warp instruction) instead of 8-byte ones.  Otherwise chunk i of every lane covers 128 consecutive columns.
template <bool PAIR>
__device__ __forceinline__ int row_col(int i, int lane) {
  return PAIR ? ((i >> 1) * 32 + lane) * 8 + (i & 1) * 4 : (i * 32 + lane) * 4;
}

// LayerNorm of a row of n columns held by the warp, in place: v[i] holds columns row_col<PAIR>(i) .. +3 (zeros past n).
// Two-pass statistics over the chunk sums (x + y) + (z + w) and fma(x, x, y y) + fma(z, z, w w), then the affine:
// FUSED_BIAS (the patch gathers, whose b is never NULL) rounds once in fma(v rstd, w, b); otherwise v * rstd * w, then + b
// when b != NULL, in LayerNorm's own expression (whether that add is contracted is the compiler's choice per instance).
template <int NV, bool PAIR, bool FUSED_BIAS>
__device__ __forceinline__ void layernorm_row(float4 (&v)[NV], int n, int lane, const float* __restrict__ w,
                                              const float* __restrict__ b, float eps) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i)
    if (row_col<PAIR>(i, lane) < n) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  const float mean = warp_sum(s) / (float)n;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    if (row_col<PAIR>(i, lane) < n) {
      v[i].x -= mean; v[i].y -= mean; v[i].z -= mean; v[i].w -= mean;
      q += fmaf(v[i].x, v[i].x, __fmul_rn(v[i].y, v[i].y)) + fmaf(v[i].z, v[i].z, __fmul_rn(v[i].w, v[i].w));
    }
  }
  const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)n + eps);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = row_col<PAIR>(i, lane);
    if (c < n) {
      const float4 g = *reinterpret_cast<const float4*>(w + c);
      float4 o;
      if constexpr (FUSED_BIAS) {
        const float4 bb = *reinterpret_cast<const float4*>(b + c);
        o.x = fmaf(__fmul_rn(v[i].x, rstd), g.x, bb.x); o.y = fmaf(__fmul_rn(v[i].y, rstd), g.y, bb.y);
        o.z = fmaf(__fmul_rn(v[i].z, rstd), g.z, bb.z); o.w = fmaf(__fmul_rn(v[i].w, rstd), g.w, bb.w);
      } else {
        o.x = v[i].x * rstd * g.x; o.y = v[i].y * rstd * g.y;
        o.z = v[i].z * rstd * g.z; o.w = v[i].w * rstd * g.w;
        if (b != nullptr) {
          const float4 bb = *reinterpret_cast<const float4*>(b + c);
          o.x += bb.x; o.y += bb.y; o.z += bb.z; o.w += bb.w;
        }
      }
      v[i] = o;
    }
  }
}

// Write a finished row of n columns (v as in layernorm_row): fp32 at out + off_f when out != NULL, and fp16 hi / lo
// planes at hi / lo + off_p when hi != NULL, row-scaled when rs != NULL (the inverse row scale to rs[row]), else 2^11-scaled.
template <int NV, bool PAIR>
__device__ __forceinline__ void store_row(const float4 (&v)[NV], int n, int lane, float* out, size_t off_f, uint16_t* hi,
                                          uint16_t* lo, size_t off_p, float* rs, int row) {
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = row_col<PAIR>(i, lane);
    if (c < n) {
      if (out != nullptr) *reinterpret_cast<float4*>(out + off_f + c) = v[i];
      if (hi != nullptr && rs == nullptr) store_split4(hi, lo, off_p + c, v[i]);
    }
  }
  if (hi != nullptr && rs != nullptr) {
    float mx = 0.f;                                    // columns past n hold zeros
#pragma unroll
    for (int i = 0; i < NV; ++i) mx = fmaxf(mx, max4abs(v[i]));
    float sc, inv;
    row_scale(warp_max(mx), sc, inv);
    if constexpr (PAIR) {
#pragma unroll
      for (int i = 0; i < NV; i += 2) {
        const int c = row_col<true>(i, lane);
        if (c < n) store_split8u(hi, lo, off_p + c, v[i], v[i + 1], sc);
      }
    } else {
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c = row_col<false>(i, lane);
        if (c < n) store_split4u(hi, lo, off_p + c, v[i], sc);
      }
    }
    if (lane == 0) rs[row] = inv;
  }
}

// ------------------------------------------------------------------------------------------
// LayerNorm: one warp per row, whole row in registers (C <= 1024), two-pass statistics.
// ------------------------------------------------------------------------------------------
struct LnPlanes {          // optional fp16 hi / lo operand planes (omt_layernorm_h), written at the LOGICAL row
  uint16_t* y_hi; uint16_t* y_lo;    // normalised row
  uint16_t* x_hi; uint16_t* x_lo;    // raw input row (Attention.forward projects k, v from it)
  int lds;
  float* y_rs; float* x_rs;          // non-NULL: row-scaled planes (omt_common.cuh), the inverse row scale goes here
};

template <int NV, bool PAIR>   // float4 chunks per lane, column map (row_col)
__global__ void __launch_bounds__(256) layernorm_kernel(const float* __restrict__ x, int ldx,
                                                        float* __restrict__ y, int ldy,
                                                        const float* __restrict__ w,
                                                        const float* __restrict__ b, int M, int C,
                                                        float eps, int seg, int seg_stride, int seg_off,
                                                        const LnPlanes pl) {
  pdl_sync();
  const int lane = threadIdx.x & 31;
  const int lrow = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (lrow >= M) return;
  const long long row = map_row(lrow, seg, seg_stride, seg_off);
  const float* xr = x + (size_t)row * ldx;
  float4 v[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = row_col<PAIR>(i, lane);
    v[i] = c < C ? *reinterpret_cast<const float4*>(xr + c) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const size_t poff = (size_t)lrow * pl.lds;
  store_row<NV, PAIR>(v, C, lane, nullptr, 0, pl.x_hi, pl.x_lo, poff, pl.x_rs, lrow);
  layernorm_row<NV, PAIR, false>(v, C, lane, w, b, eps);
  store_row<NV, PAIR>(v, C, lane, y, (size_t)row * ldy, pl.y_hi, pl.y_lo, poff, pl.y_rs, lrow);
}

// ------------------------------------------------------------------------------------------
// Patch gather + LayerNorm.  One warp per patch row; K = Cin*p*p (first frame) or Cin*pt*p*p.
// Feature f = ((c*PT + dt)*p + p1)*p + p2 ; p2 is contiguous in the video (p % 4 == 0).
// The gather (fp32 video or uint8 frames) fills the lane's v[i] = features f = row_col<false>(i) .. +3 (zeros past K);
// patch_ln_emit() is the LayerNorm and output stage both gathers share, so equal v[] give equal bits.
// ------------------------------------------------------------------------------------------
struct PatchRow {             // patch row -> (sample, first frame of the row, token row / column)
  int bi, t0, hi, wi;
};

__device__ __forceinline__ PatchRow patch_row(int row, int T, int H, int W, int p, int pt, int first) {
  const int hh = H / p, ww = W / p;
  int r = row;
  PatchRow pr;
  pr.wi = r % ww; r /= ww;
  pr.hi = r % hh; r /= hh;
  int ti = 0;
  if (!first) { const int tn = (T - 1) / pt; ti = r % tn; r /= tn; }
  pr.bi = r;
  pr.t0 = first ? 0 : 1 + ti * pt;
  return pr;
}

struct PatchFeature {         // feature f of a patch row -> (channel, frame in the patch, patch row / column)
  int c, dt, p1, p2;
};

__device__ __forceinline__ PatchFeature patch_feature(int f, int p, int PT) {
  PatchFeature pf;
  pf.p2 = f % p;
  pf.p1 = (f / p) % p;
  pf.dt = (f / (p * p)) % PT;
  pf.c = f / (p * p * PT);
  return pf;
}

// Element of feature pf of patch row pr in the (B, Cin, T, H, W) video.
__device__ __forceinline__ size_t patch_elem(const PatchRow& pr, const PatchFeature& pf, int Cin, int T, int H, int W, int p) {
  return ((((size_t)pr.bi * Cin + pf.c) * T + (pr.t0 + pf.dt)) * H + (pr.hi * p + pf.p1)) * W + pr.wi * p + pf.p2;
}

template <int NV>
__device__ __forceinline__ void patch_ln_emit(float4 (&v)[NV], int row, int K, int lane, float* __restrict__ A,
                                              uint16_t* __restrict__ A_hi, uint16_t* __restrict__ A_lo,
                                              float* __restrict__ A_rs, const float* __restrict__ lw,
                                              const float* __restrict__ lb, float eps) {
  // lw == NULL: plain im2col (patch_embed='cnn': the strided Conv3d is a GEMM on raw patch vectors)
  if (lw != nullptr) layernorm_row<NV, false, true>(v, K, lane, lw, lb, eps);
  const size_t off = (size_t)row * K;
  store_row<NV, false>(v, K, lane, A_hi != nullptr ? nullptr : A, off, A_hi, A_lo, off, A_rs, row);   // planes replace A
}

template <int NV>
__global__ void __launch_bounds__(256) patchify_ln_kernel(const float* __restrict__ video,
                                                          float* __restrict__ A, uint16_t* __restrict__ A_hi,
                                                          uint16_t* __restrict__ A_lo, float* __restrict__ A_rs,
                                                          const float* __restrict__ lw,
                                                          const float* __restrict__ lb, int rows,
                                                          int Cin, int T, int H, int W, int p, int pt,
                                                          int first, float eps) {
  pdl_sync();
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int PT = first ? 1 : pt;
  const int K = Cin * PT * p * p;
  const PatchRow pr = patch_row(row, T, H, W, p, pt, first);
  float4 v[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int f = row_col<false>(i, lane);
    v[i] = f < K ? *reinterpret_cast<const float4*>(video + patch_elem(pr, patch_feature(f, p, PT), Cin, T, H, W, p))
                 : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  patch_ln_emit<NV>(v, row, K, lane, A, A_hi, A_lo, A_rs, lw, lb, eps);
}

// uint8 twin: frames (B, T, H, W, Cin) channels-last bytes, each byte of channel c mapped through lut[tab][c][256], the
// host-built table of the data pipeline's normalisation (tab = sel[b], or 0 without sel).  A patch line of one row is p*Cin
// contiguous, 4-byte aligned bytes: each warp stages its row's PT*p lines in shared memory with 32-bit loads, then builds
// the same v[] as patchify_ln_kernel.  Warps walk rows with a grid stride so the table is loaded once per CTA.
constexpr int PU8_WARPS = 8;
constexpr int PATCH_MAX_K = 1024;   // longest patch vector of both gathers: 8 float4 chunks per lane; the bytes of one staged row

template <int NV>
__global__ void __launch_bounds__(256) patchify_ln_u8_kernel(const uint8_t* __restrict__ frames,
                                                             const float* __restrict__ lut, const int32_t* __restrict__ sel,
                                                             float* __restrict__ A, uint16_t* __restrict__ A_hi,
                                                             uint16_t* __restrict__ A_lo, float* __restrict__ A_rs,
                                                             const float* __restrict__ lw, const float* __restrict__ lb,
                                                             int rows, int Cin, int T, int H, int W, int p, int pt,
                                                             int first, float eps) {
  __shared__ float tab[2 * 4 * 256];
  __shared__ uint32_t stage[PU8_WARPS][PATCH_MAX_K / 4];
  pdl_sync();
  const int ntab = sel != nullptr ? 2 : 1;
  for (int i = threadIdx.x; i < ntab * Cin * 256; i += blockDim.x) tab[i] = lut[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int PT = first ? 1 : pt;
  const int K = Cin * PT * p * p;
  const int line_words = p * Cin / 4;
  uint32_t* st = stage[warp];
  const uint8_t* sb = reinterpret_cast<const uint8_t*>(st);
  for (int row = blockIdx.x * PU8_WARPS + warp; row < rows; row += gridDim.x * PU8_WARPS) {
    const PatchRow pr = patch_row(row, T, H, W, p, pt, first);
    for (int j = lane; j < K / 4; j += 32) {          // word j of line l = dt * p + p1
      const int l = j / line_words;
      const int dt = l / p, p1 = l - dt * p;
      const size_t pix = (((size_t)pr.bi * T + (pr.t0 + dt)) * H + (pr.hi * p + p1)) * W + pr.wi * p;
      st[j] = __ldg(reinterpret_cast<const uint32_t*>(frames + pix * Cin) + (j - l * line_words));
    }
    __syncwarp();
    const float* tb = tab;
    if (sel != nullptr) tb += (sel[pr.bi] != 0 ? Cin * 256 : 0);
    float4 v[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int f = row_col<false>(i, lane);
      if (f < K) {
        const PatchFeature pf = patch_feature(f, p, PT);
        const uint8_t* px = sb + ((pf.dt * p + pf.p1) * p + pf.p2) * Cin + pf.c;
        const float* tc = tb + pf.c * 256;
        v[i] = make_float4(tc[px[0]], tc[px[Cin]], tc[px[2 * Cin]], tc[px[3 * Cin]]);
      } else {
        v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    __syncwarp();                                      // the stage is rewritten by the next row
    patch_ln_emit<NV>(v, row, K, lane, A, A_hi, A_lo, A_rs, lw, lb, eps);
  }
}

// sel[b] = 1 until a byte > 1 is found in sample b (VideoNorm's `if max(clip) > 1: div_(255)`), then 0.
__global__ void __launch_bounds__(256) u8_sel_init_kernel(int32_t* __restrict__ sel, int B) {
  pdl_sync();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) sel[b] = 1;
}

__global__ void __launch_bounds__(256) u8_sel_scan_kernel(const uint8_t* __restrict__ frames, long long per_sample,
                                                          int32_t* __restrict__ sel) {
  pdl_sync();
  const uint8_t* x = frames + (size_t)blockIdx.y * per_sample;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long t0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t acc = 0;
  if (per_sample % 16 == 0 && (reinterpret_cast<uintptr_t>(frames) & 15) == 0) {
    const uint4* x4 = reinterpret_cast<const uint4*>(x);
    for (long long i = t0; i < per_sample / 16; i += stride) {
      const uint4 w = __ldg(x4 + i);
      acc |= w.x | w.y | w.z | w.w;
    }
  } else {
    for (long long i = t0; i < per_sample; i += stride) acc |= x[i];
  }
  // a byte is > 1 exactly when one of its bits 1..7 is set
  if (__syncthreads_or((acc & 0xFEFEFEFEu) != 0) && threadIdx.x == 0) sel[blockIdx.y] = 0;
}

__global__ void __launch_bounds__(256) unpatchify_kernel(const float* __restrict__ P,
                                                         float* __restrict__ video, long long total4,
                                                         int Cin, int T, int H, int W, int p, int pt,
                                                         int first) {
  pdl_sync();
  const int PT = first ? 1 : pt;
  const int K4 = Cin * PT * p * p / 4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total4;
       i += (long long)gridDim.x * blockDim.x) {
    const PatchRow pr = patch_row((int)(i / K4), T, H, W, p, pt, first);
    const PatchFeature pf = patch_feature((int)(i % K4) * 4, p, PT);
    *reinterpret_cast<float4*>(video + patch_elem(pr, pf, Cin, T, H, W, p)) = *reinterpret_cast<const float4*>(P + i * 4);
  }
}

// ------------------------------------------------------------------------------------------
// Un-patchify fused with the consumer's uint8 conversion (vqgan_eval.py:139,147-148; Latte sample_ddp.py:206;
// DiT sample_ddp.py:163):  u8 = trunc( clamp(x * mul + add, lo, hi) * post )  written channels-LAST
// (b, t, H, W, c) -- the layout every consumer permutes to before .byte().  mul / add / post are applied as separate
// fp32 roundings (no fma contraction) so the bytes equal torch's elementwise expression on the fp32 reconstruction.
// One thread = 4 consecutive pixels of one patch line, all Cin channels (Cin * 4 bytes contiguous in the output).
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) unpatchify_u8_kernel(const float* __restrict__ P, uint8_t* __restrict__ out,
                                                            long long total, int Cin, int T, int H, int W, int p,
                                                            int pt, int first, float mul, float add, float lo,
                                                            float hi, float post) {
  pdl_sync();
  const int PT = first ? 1 : pt;
  const int per_row = PT * p * (p / 4);           // (dt, p1, p2-quad) items per patch row
  const int K = Cin * PT * p * p;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    int it = (int)(i % per_row);
    const int row = (int)(i / per_row);
    const int q4 = it % (p / 4); it /= (p / 4);
    const int p1 = it % p;
    const int dt = it / p;
    const PatchRow pr = patch_row(row, T, H, W, p, pt, first);
    const size_t pix = (((size_t)pr.bi * T + (pr.t0 + dt)) * H + (pr.hi * p + p1)) * W + pr.wi * p + q4 * 4;
    uint8_t* o = out + pix * Cin;
    for (int c = 0; c < Cin; ++c) {
      const float4 v = *reinterpret_cast<const float4*>(P + (size_t)row * K + ((c * PT + dt) * p + p1) * p + q4 * 4);
      const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float tv = __fadd_rn(__fmul_rn(e[j], mul), add);
        tv = fminf(fmaxf(tv, lo), hi);
        o[j * Cin + c] = (uint8_t)__float2uint_rz(__fmul_rn(tv, post));
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// PEG: y = x + bias + sum_k w[k] * x[nbr[k]].  Block = C/4 threads (one float4 channel group
// each), loops over ROWS consecutive rows; the 27 x C weight table sits in shared memory.
// ------------------------------------------------------------------------------------------
constexpr int PEG_ROWS = 16;

__global__ void __launch_bounds__(128) peg_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                  const float* __restrict__ w27,
                                                  const float* __restrict__ bias,
                                                  const int32_t* __restrict__ nbr, int rows_per_b,
                                                  int C, long long M) {
  pdl_sync();
  extern __shared__ float4 wsm[];   // [27][C/4]
  __shared__ int32_t nsm[PEG_ROWS][27];
  const int c4 = threadIdx.x;       // channel group
  const int C4 = C >> 2;
  for (int i = threadIdx.x; i < 27 * C4; i += blockDim.x)
    wsm[i] = reinterpret_cast<const float4*>(w27)[i];
  const long long r0 = (long long)blockIdx.x * PEG_ROWS;
  for (int i = threadIdx.x; i < PEG_ROWS * 27; i += blockDim.x) {
    const long long r = r0 + i / 27;
    nsm[i / 27][i % 27] = (r < M) ? nbr[(r % rows_per_b) * 27 + (i % 27)] : -1;
  }
  __syncthreads();
  if (c4 >= C4) return;
  const float4 bb = reinterpret_cast<const float4*>(bias)[c4];
  for (int rr = 0; rr < PEG_ROWS; ++rr) {
    const long long r = r0 + rr;
    if (r >= M) break;
    const long long base = (r / rows_per_b) * rows_per_b;
    const float4 xv = reinterpret_cast<const float4*>(x + r * C)[c4];
    float4 acc = bb;
#pragma unroll
    for (int k = 0; k < 27; ++k) {
      const int n = nsm[rr][k];
      if (n >= 0) {
        const float4 nv = __ldg(reinterpret_cast<const float4*>(x + (base + n) * C) + c4);
        const float4 wv = wsm[k * C4 + c4];
        acc.x = fmaf(nv.x, wv.x, acc.x); acc.y = fmaf(nv.y, wv.y, acc.y);
        acc.z = fmaf(nv.z, wv.z, acc.z); acc.w = fmaf(nv.w, wv.w, acc.w);
      }
    }
    acc.x += xv.x; acc.y += xv.y; acc.z += xv.z; acc.w += xv.w;
    reinterpret_cast<float4*>(y + r * C)[c4] = acc;
  }
}

// ------------------------------------------------------------------------------------------
// PEG, tiled form.  The stencil lives in "volume space" (t2,h2,w2): for spatial transformers that
// is the true token grid; for temporal ones it is the reference's literal reshape of the
// '(b h w) t d' tensor (flat f = n*T + tau unravelled over (T,h,w)).  Either way volume position f
// maps to canonical row  temporal ? (f % T) * N + f / T : f.
// One CTA stages a (TT+2) x (HB+2) x (w+2) x 16-channel halo tile in shared memory (zeros where the
// reference pads), then every thread owns one (plane, row, channel-pair) strip and slides a
// 3x3x3 register window along w: 9 shared loads per output instead of 27 global ones.
// ------------------------------------------------------------------------------------------
constexpr int PEG_CC = 16;       // channels per CTA

__global__ void __launch_bounds__(256) peg_tile_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                       const float* __restrict__ w27,
                                                       const float* __restrict__ bias, int T, int h, int w,
                                                       int C, int temporal, int causal, int TT, int HB, int RS,
                                                       const int32_t* __restrict__ t_off) {
  pdl_sync();
  extern __shared__ __align__(16) float tile[];      // [(TT+2)][(HB+2)] rows of RS floats ((w+2)*16 + pad)
  const int N = h * w;
  const int n_hblk = (h + HB - 1) / HB;
  const int t0 = (blockIdx.x / n_hblk) * TT, h0 = (blockIdx.x % n_hblk) * HB;
  const int c0 = blockIdx.y * PEG_CC;
  long long bbase = (long long)blockIdx.z * T * N;
  if (t_off != nullptr) {                            // packed batch: this sample's own T' and rows (T = the longest)
    const int f0 = t_off[blockIdx.z];
    T = t_off[blockIdx.z + 1] - f0;
    bbase = (long long)f0 * N;
    if (t0 >= T) return;
  }
  const int pad_lo = causal ? 2 : 1;
  const int rows = (TT + 2) * (HB + 2);
  const int nth = blockDim.x;
  // ---- halo tile: the (few) integer divisions happen once per (plane,row) pair and once per position,
  //      not once per 16-byte load: int2 {global row or -1, smem float offset} per position
  int2* pmap = reinterpret_cast<int2*>(tile + rows * RS);
  const int P = rows * (w + 2);
  for (int pos = threadIdx.x; pos < P; pos += nth) {
    const int pw = pos % (w + 2);
    const int pr = pos / (w + 2);
    const int ph = pr % (HB + 2), pt = pr / (HB + 2);
    const int t2 = t0 - pad_lo + pt, h2 = h0 - 1 + ph, w2 = pw - 1;
    int row = -1;
    if (t2 >= 0 && t2 < T && h2 >= 0 && h2 < h && w2 >= 0 && w2 < w) {
      const int f = (t2 * h + h2) * w + w2;
      row = temporal ? (f % T) * N + f / T : f;
    }
    pmap[pos] = make_int2(row, pr * RS + pw * PEG_CC);
  }
  __syncthreads();
  // gathers are issued in batches of 8 per thread before any shared store so ~8 x 16 B are in flight per thread
  for (int i0 = threadIdx.x; i0 < P * 4; i0 += nth * 8) {
    float4 v[8];
    int so[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int i = i0 + u * nth;
      v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      so[u] = -1;
      if (i < P * 4) {
        const int2 pm = pmap[i >> 2];
        so[u] = pm.y + (i & 3) * 4;
        if (pm.x >= 0) v[u] = __ldg(reinterpret_cast<const float4*>(x + (bbase + pm.x) * C + c0) + (i & 3));
      }
    }
#pragma unroll
    for (int u = 0; u < 8; ++u)
      if (so[u] >= 0) *reinterpret_cast<float4*>(tile + so[u]) = v[u];
  }
  __syncthreads();
  // ---- strips
  const int cp = threadIdx.x & 7;                  // channel pair inside the 16-channel slab
  const int strip = threadIdx.x >> 3;
  const int sh = strip % HB, st = strip / HB;
  if (st >= TT || t0 + st >= T || h0 + sh >= h) return;
  float2 wt[27];
#pragma unroll
  for (int k = 0; k < 27; ++k) wt[k] = *reinterpret_cast<const float2*>(w27 + (size_t)k * C + c0 + 2 * cp);
  const float2 bb = *reinterpret_cast<const float2*>(bias + c0 + 2 * cp);
  float2 win[9][3];
  const float* tp = tile + 2 * cp;
#pragma unroll
  for (int r9 = 0; r9 < 9; ++r9) {
    const float* rp = tp + ((st + r9 / 3) * (HB + 2) + sh + r9 % 3) * RS;
    win[r9][1] = *reinterpret_cast<const float2*>(rp);
    win[r9][2] = *reinterpret_cast<const float2*>(rp + PEG_CC);
  }
  const int fbase = ((t0 + st) * h + (h0 + sh)) * w;
  int tau = fbase % T, nn = fbase / T;               // temporal: volume position f <-> canonical (tau, n), advanced incrementally
  for (int w2 = 0; w2 < w; ++w2) {
    float2 acc = bb;
#pragma unroll
    for (int r9 = 0; r9 < 9; ++r9) {
      const float* rp = tp + ((st + r9 / 3) * (HB + 2) + sh + r9 % 3) * RS + (w2 + 2) * PEG_CC;
      win[r9][0] = win[r9][1]; win[r9][1] = win[r9][2];
      win[r9][2] = *reinterpret_cast<const float2*>(rp);
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        acc.x = fmaf(win[r9][kw].x, wt[r9 * 3 + kw].x, acc.x);
        acc.y = fmaf(win[r9][kw].y, wt[r9 * 3 + kw].y, acc.y);
      }
    }
    const float2 ctr = causal ? win[7][1] : win[4][1];   // the un-shifted token itself (residual)
    acc.x += ctr.x; acc.y += ctr.y;
    const int row = temporal ? tau * N + nn : fbase + w2;
    *reinterpret_cast<float2*>(y + (bbase + row) * C + c0 + 2 * cp) = acc;
    if (++tau == T) { tau = 0; ++nn; }
  }
}

// ------------------------------------------------------------------------------------------
// PEG, tiled form v4: same tile geometry and the SAME fma order as peg_tile_kernel (bit-identical output), with
// the instruction count cut ~3x (the v3 kernel is issue-bound: ncu 67 M warp instructions, 102 per output):
//   * halo gather by cp.async (16 B, zero-fill where the reference pads): no register staging, no position-map
//     pass; one warp walks one halo row at a time so the only divisions are per row (warp-uniform) and the
//     temporal  f -> (f % T, f / T)  split is a multiply-shift on the in-row offset;
//   * the 3x3x3 register window rotates by renaming (w loop unrolled by 3) instead of 36 MOVs per output;
//   * channel pairs (float2) per thread: one 8-byte shared-memory load per pair and tap.
// Requires T <= 64 and w <= 254 (multiply-shift range); the host falls back to v3 otherwise (x is 16-byte aligned for both).
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float2 lds_f2(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
  return v;
}
// One output position of a strip.  R = window rotation: tap kw of window row r9 lives in slot (kw + R) % 3;
// the new halo column is read at a[r9] + R * 64 bytes (a[] points at the trip's first new column).
template <int R>
__device__ __forceinline__ float2 peg_step(float2 (&win)[9][3], const float2 (&wt)[27], const float2 bb,
                                           const uint32_t (&a)[9], const bool causal) {
  float2 acc = bb;
#pragma unroll
  for (int r9 = 0; r9 < 9; ++r9) {
    win[r9][(2 + R) % 3] = lds_f2(a[r9] + R * (PEG_CC * 4));
#pragma unroll
    for (int kw = 0; kw < 3; ++kw) acc = ffma2(win[r9][(kw + R) % 3], wt[r9 * 3 + kw], acc);
  }
  const float2 ctr = causal ? win[7][(1 + R) % 3] : win[4][(1 + R) % 3];   // the un-shifted token itself (residual)
  acc.x += ctr.x; acc.y += ctr.y;
  return acc;
}

__global__ void __launch_bounds__(160, 3) peg_tile4_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                           const float* __restrict__ w27,
                                                           const float* __restrict__ bias, int T, int h, int w,
                                                           int C, int temporal, int causal, int TT, int HB, int RS, int zrow,
                                                           const int32_t* __restrict__ t_off) {
  pdl_sync();
  // [valid planes of the tile][(HB+2)] rows of RS floats ((w+2)*16 + pad), then ONE all-zero row at index zrow: planes
  // outside the volume (the causal pad in front, the halo behind the last plane) are not stored -- every window row that
  // falls into one reads the zero row instead.  5 of 7 planes at T' = 5: 69 KB instead of 94 KB, three CTAs per SM.
  extern __shared__ __align__(16) float tile[];
  const int N = h * w;
  const int n_hblk = (h + HB - 1) / HB;
  const int t0 = (blockIdx.x / n_hblk) * TT, h0 = (blockIdx.x % n_hblk) * HB;
  const int c0 = blockIdx.y * PEG_CC;
  long long bbase = (long long)blockIdx.z * T * N;
  if (t_off != nullptr) {                            // packed batch: this sample's own T' and rows (T = the longest)
    const int f0 = t_off[blockIdx.z];
    T = t_off[blockIdx.z + 1] - f0;
    bbase = (long long)f0 * N;
    if (t0 >= T) return;
  }
  const int pad_lo = causal ? 2 : 1;
  const int rows = (TT + 2) * (HB + 2);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const uint32_t inv_T = (65536u + (uint32_t)T - 1u) / (uint32_t)T;       // floor(v / T) == (v * inv_T) >> 16 for v < 65536 / T
  const uint32_t tile_s = static_cast<uint32_t>(__cvta_generic_to_shared(tile));
  const int chunks = (w + 2) * 4;                                          // 16-byte chunks per halo row
  const int pz_lo = t0 < pad_lo ? pad_lo - t0 : 0;                         // leading planes of the tile that lie before t = 0
  for (int i = threadIdx.x; i < RS / 4; i += blockDim.x)
    asm volatile("st.shared.v4.f32 [%0], {%1, %1, %1, %1};" ::"r"(tile_s + (uint32_t)(zrow * RS + 4 * i) * 4u), "f"(0.f) : "memory");
  // ---- halo tile: warp <-> halo row; lane <-> 16-byte chunk (consecutive lanes write consecutive shared addresses)
  for (int pr = warp; pr < rows; pr += nwarps) {
    const int ph = pr % (HB + 2), pt = pr / (HB + 2);
    const int t2 = t0 - pad_lo + pt, h2 = h0 - 1 + ph;
    if (t2 < 0 || t2 >= T) continue;                                       // plane outside the volume: not stored
    const bool row_ok = h2 >= 0 && h2 < h;
    const int fb = row_ok ? (t2 * h + h2) * w : 0;                         // volume position of (t2, h2, w2 = 0)
    const int tau0 = fb % T, nn0 = fb / T;
    const uint32_t dst_row = tile_s + (uint32_t)(((pt - pz_lo) * (HB + 2) + ph) * RS) * 4u;
    for (int j = lane; j < chunks; j += 32) {
      const int w2 = (j >> 2) - 1;
      const bool ok = row_ok && w2 >= 0 && w2 < w;
      long long row = 0;
      if (ok) {
        if (temporal) {
          const uint32_t v = (uint32_t)(tau0 + w2);
          const uint32_t q = (v * inv_T) >> 16;
          row = (long long)(v - q * (uint32_t)T) * N + nn0 + (int)q;
        } else {
          row = fb + w2;
        }
      }
      const float* src = x + (bbase + row) * C + c0 + (j & 3) * 4;
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst_row + (uint32_t)j * 16u), "l"(src), "r"(ok ? 16 : 0) : "memory");
    }
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
  // ---- strips: weights are fetched while the gather is in flight
  const int cp = threadIdx.x & 7;                  // channel pair inside the 16-channel slab
  const int strip = threadIdx.x >> 3;
  const int sh = strip % HB, st = strip / HB;
  const bool active = st < TT && t0 + st < T && h0 + sh < h;
  float2 wt[27];
  float2 bb = make_float2(0.f, 0.f);
  if (active) {
#pragma unroll
    for (int k = 0; k < 27; ++k) wt[k] = __ldg(reinterpret_cast<const float2*>(w27 + (size_t)k * C + c0 + 2 * cp));
    bb = __ldg(reinterpret_cast<const float2*>(bias + c0 + 2 * cp));
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncthreads();
  if (!active) return;
  // shared byte addresses of halo column 0 of the 9 window rows of this strip
  uint32_t a[9];
#pragma unroll
  for (int r9 = 0; r9 < 9; ++r9) {
    const int pt = st + r9 / 3;                     // tile plane of this window row
    const int t2 = t0 - pad_lo + pt;
    const int prow = (t2 < 0 || t2 >= T) ? zrow : (pt - pz_lo) * (HB + 2) + sh + r9 % 3;
    a[r9] = tile_s + (uint32_t)((prow * RS + 2 * cp) * 4);
  }
  float2 win[9][3];
#pragma unroll
  for (int r9 = 0; r9 < 9; ++r9) {
    win[r9][0] = lds_f2(a[r9]);                     // halo column 0 (w2 = -1)
    win[r9][1] = lds_f2(a[r9] + PEG_CC * 4);        // halo column 1 (w2 = 0)
    a[r9] += 2 * PEG_CC * 4;                        // -> the first new column of trip 0 (halo column 2)
  }
  // output pointer, advanced incrementally: spatial rows are consecutive; temporal rows follow the literal
  // reshape  f -> (tau, n) = (f % T, f / T)  ->  canonical row tau * N + n
  const int fbase = ((t0 + st) * h + (h0 + sh)) * w;
  int tau = fbase % T;
  const long long row0 = temporal ? (long long)tau * N + fbase / T : (long long)fbase;
  float* yp = y + (bbase + row0) * C + c0 + 2 * cp;
  const long long inc = temporal ? (long long)N * C : (long long)C;
  const long long wrap = (long long)T * N * C - C;   // temporal: tau T-1 -> 0 moves back T planes and on one token
  const bool cz = causal != 0;
#define OMT_PEG_STEP(R)                                                                             \
  {                                                                                                 \
    const float2 acc = peg_step<R>(win, wt, bb, a, cz);                                             \
    *reinterpret_cast<float2*>(yp) = acc;                                                           \
    yp += inc;                                                                                      \
    if (temporal && ++tau == T) { tau = 0; yp -= wrap; }                                            \
  }
  for (int wb = 0; wb < w; wb += 3) {
    OMT_PEG_STEP(0)
    if (wb + 1 < w) OMT_PEG_STEP(1)
    if (wb + 2 < w) OMT_PEG_STEP(2)
#pragma unroll
    for (int r9 = 0; r9 < 9; ++r9) a[r9] += 3 * PEG_CC * 4;
  }
#undef OMT_PEG_STEP
}

// ------------------------------------------------------------------------------------------
// rope + l2norm + scale, in place on q and k.  One warp per row; lane l owns the complex pair
// (2l, 2l+1) of every head.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void qk_prep_one(float* p, const float2 cs, bool rope, const float2 sc) {
  float2 v = *reinterpret_cast<float2*>(p);
  if (rope) {
    const float a = v.x * cs.x - v.y * cs.y;
    const float b = v.x * cs.y + v.y * cs.x;
    v.x = a; v.y = b;
  }
  const float ss = warp_sum(v.x * v.x + v.y * v.y);
  const float den = fmaxf(sqrtf(ss), 1e-12f);
  v.x = v.x / den * sc.x;
  v.y = v.y / den * sc.y;
  *reinterpret_cast<float2*>(p) = v;
}

__global__ void __launch_bounds__(256) qk_prep_kernel(float* __restrict__ q, int ldq,
                                                      float* __restrict__ k, int ldk,
                                                      const float* __restrict__ qs,
                                                      const float* __restrict__ ks,
                                                      const float* __restrict__ rc,
                                                      const float* __restrict__ rs, int M, int N,
                                                      int heads) {
  pdl_sync();
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= M) return;
  const bool rope = rc != nullptr;
  float2 cs = make_float2(1.f, 0.f);
  if (rope) {
    const int pos = row % N;
    cs.x = rc[pos * 32 + lane];
    cs.y = rs[pos * 32 + lane];
  }
  const float2 sq = *reinterpret_cast<const float2*>(qs + 2 * lane);
  const float2 sk = *reinterpret_cast<const float2*>(ks + 2 * lane);
  for (int h = 0; h < heads; ++h) {
    qk_prep_one(q + (size_t)row * ldq + h * 64 + 2 * lane, cs, rope, sq);
    qk_prep_one(k + (size_t)row * ldk + h * 64 + 2 * lane, cs, rope, sk);
  }
}

}  // namespace omt

using namespace omt;

static int layernorm_impl(const char* who, const float* x, int ldx, float* y, int ldy, const omt::LnPlanes& pl, const float* w,
                          const float* b, int M, int C, float eps, int seg, int seg_stride, int seg_off, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(x && w && (y || pl.y_hi), "%s: null pointer", who);
  OMT_REQUIRE(M >= 0 && C > 0 && C % 4 == 0 && C <= 1024, "%s: C=%d must be a multiple of 4, <= 1024", who, C);
  OMT_REQUIRE(ldx % 4 == 0 && ldx >= C && (y == nullptr || (ldy % 4 == 0 && ldy >= C)), "%s: bad leading dims", who);
  OMT_REQUIRE(aligned_to(16, {x, y, w, b}), "%s: x, y, w and b must be 16-byte aligned", who);
  OMT_REQUIRE((pl.y_hi == nullptr) == (pl.y_lo == nullptr) && (pl.x_hi == nullptr) == (pl.x_lo == nullptr), "%s: planes come in hi / lo pairs", who);
  if (pl.y_hi != nullptr || pl.x_hi != nullptr) {
    OMT_REQUIRE(pl.lds % 4 == 0 && pl.lds >= C, "%s: plane leading dimension %d", who, pl.lds);
    OMT_REQUIRE(((uintptr_t)pl.y_hi | (uintptr_t)pl.y_lo | (uintptr_t)pl.x_hi | (uintptr_t)pl.x_lo) % 8 == 0, "%s: planes must be 8-byte aligned", who);
  }
  if (M == 0) return OMT_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int nv = (C / 4 + 31) / 32;
  // 8 consecutive columns per lane (16-byte plane stores) when the row splits into whole 256-column blocks and the planes allow it
  const bool pair = C % 256 == 0 && pl.lds % 8 == 0 &&
                    ((uintptr_t)pl.y_hi | (uintptr_t)pl.y_lo | (uintptr_t)pl.x_hi | (uintptr_t)pl.x_lo) % 16 == 0;
  // PAIR implies C = 128 NV with NV = 2, 4, 6 or 8; unpaired widths of more than 4 chunks take <8, false>
  using LnKernel = decltype(&layernorm_kernel<1, false>);
  static const LnKernel paired[] = {layernorm_kernel<2, true>, layernorm_kernel<4, true>, layernorm_kernel<6, true>,
                                    layernorm_kernel<8, true>};
  static const LnKernel unpaired[] = {layernorm_kernel<1, false>, layernorm_kernel<2, false>, layernorm_kernel<3, false>,
                                      layernorm_kernel<4, false>};
  const LnKernel kernel = pair ? paired[nv / 2 - 1] : (nv <= 4 ? unpaired[nv - 1] : layernorm_kernel<8, false>);
  OMT_CUDA(launch_k(kernel, dim3((M + 7) / 8), dim3(256), 0, st, x, ldx, y, ldy, w, b, M, C, eps, seg, seg_stride, seg_off, pl));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

extern "C" int omt_layernorm(const float* x, int ldx, float* y, int ldy, const float* w, const float* b,
                             int M, int C, float eps, int seg, int seg_stride, int seg_off,
                             omt_stream_t stream) {
  OMT_REQUIRE(y != nullptr, "omt_layernorm: null pointer");
  omt::LnPlanes pl{nullptr, nullptr, nullptr, nullptr, 0, nullptr, nullptr};
  return layernorm_impl("omt_layernorm", x, ldx, y, ldy, pl, w, b, M, C, eps, seg, seg_stride, seg_off, stream);
}

extern "C" int omt_layernorm_h(const float* x, int ldx, float* y, int ldy, uint16_t* y_hi, uint16_t* y_lo, float* y_rs,
                               uint16_t* x_hi, uint16_t* x_lo, float* x_rs, int lds, const float* w, const float* b,
                               int M, int C, float eps, int seg, int seg_stride, int seg_off, omt_stream_t stream) {
  OMT_REQUIRE((y_rs == nullptr || y_hi != nullptr) && (x_rs == nullptr || x_hi != nullptr), "omt_layernorm_h: row scales without planes");
  omt::LnPlanes pl{y_hi, y_lo, x_hi, x_lo, lds, y_rs, x_rs};
  return layernorm_impl("omt_layernorm_h", x, ldx, y, ldy, pl, w, b, M, C, eps, seg, seg_stride, seg_off, stream);
}

// Patch geometry of the four patch entry points: a (B, Cin, T, H, W) video cut into p x p patches of the first frame
// (first) or of pt frames from frame 1 on.  The checks run in this order so that no division meets an unchecked divisor.
// *rows = patch rows, *K = features per row.
static int check_patch_geometry(const char* who, int B, int Cin, int T, int H, int W, int p, int pt, int first,
                                long long* rows, int* K) {
  OMT_REQUIRE(B >= 0, "%s: B=%d", who, B);
  OMT_REQUIRE(Cin >= 1, "%s: Cin=%d must be >= 1", who, Cin);
  OMT_REQUIRE(p > 0 && p % 4 == 0 && H % p == 0 && W % p == 0, "%s: patch %d must be a positive multiple of 4 dividing %dx%d",
              who, p, H, W);
  OMT_REQUIRE(first || (T > 1 && pt > 0 && (T - 1) % pt == 0), "%s: (T-1) %% pt != 0 or pt <= 0 (T=%d, pt=%d)", who, T, pt);
  *K = Cin * (first ? 1 : pt) * p * p;
  *rows = (long long)B * (first ? 1 : (T - 1) / pt) * (H / p) * (W / p);
  return OMT_OK;
}

// Arguments both gathers check alike: the outputs (A, or hi / lo planes, with row scales only beside planes), LayerNorm
// weights both or neither, the patch geometry and the patch vector's length.
static int check_gather(const char* who, const float* A, const uint16_t* A_hi, const uint16_t* A_lo, const float* A_rs,
                        const float* ln_w, const float* ln_b, int B, int Cin, int T, int H, int W, int p, int pt, int first,
                        long long* rows, int* K) {
  OMT_REQUIRE((A || A_hi) && (ln_w == nullptr) == (ln_b == nullptr) && (A_hi == nullptr) == (A_lo == nullptr),
              "%s: null pointer", who);
  OMT_REQUIRE(A_rs == nullptr || A_hi != nullptr, "%s: row scales without planes", who);
  OMT_REQUIRE(aligned_to(16, {A, ln_w, ln_b}), "%s: A, ln_w and ln_b must be 16-byte aligned", who);
  OMT_REQUIRE(aligned_to(8, {A_hi, A_lo}), "%s: planes must be 8-byte aligned", who);
  const int rc = check_patch_geometry(who, B, Cin, T, H, W, p, pt, first, rows, K);
  if (rc != OMT_OK) return rc;
  OMT_REQUIRE(*K <= PATCH_MAX_K, "%s: patch vector %d > %d", who, *K, PATCH_MAX_K);
  return OMT_OK;
}

// float4 chunks per lane of both gathers: 2, 6 or 8 (entry 0, 1 or 2 of their kernel tables)
static int gather_nv_index(int K) {
  const int nv = (K / 4 + 31) / 32;
  return nv <= 2 ? 0 : (nv <= 6 ? 1 : 2);
}

extern "C" int omt_patchify_ln(const float* video, float* A, uint16_t* A_hi, uint16_t* A_lo, float* A_rs, const float* ln_w,
                               const float* ln_b, int B, int Cin, int T, int H, int W, int p, int pt, int first,
                               float eps, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(video, "omt_patchify_ln: null pointer");
  OMT_REQUIRE(aligned_to(16, {video}), "omt_patchify_ln: video must be 16-byte aligned");
  long long rows;
  int K;
  const int rc = check_gather("omt_patchify_ln", A, A_hi, A_lo, A_rs, ln_w, ln_b, B, Cin, T, H, W, p, pt, first, &rows, &K);
  if (rc != OMT_OK) return rc;
  if (rows == 0) return OMT_OK;
  static decltype(&patchify_ln_kernel<2>) const kernels[] = {patchify_ln_kernel<2>, patchify_ln_kernel<6>, patchify_ln_kernel<8>};
  OMT_CUDA(launch_k(kernels[gather_nv_index(K)], dim3((unsigned)((rows + 7) / 8)), dim3(256), 0, (cudaStream_t)stream, video,
                    A, A_hi, A_lo, A_rs, ln_w, ln_b, (int)rows, Cin, T, H, W, p, pt, first, eps));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

extern "C" int omt_patchify_ln_u8(const uint8_t* frames, const float* lut, const int32_t* sel, float* A, uint16_t* A_hi,
                                  uint16_t* A_lo, float* A_rs, const float* ln_w, const float* ln_b, int B, int Cin, int T,
                                  int H, int W, int p, int pt, int first, float eps, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(frames && lut, "omt_patchify_ln_u8: null pointer");
  OMT_REQUIRE(aligned_to(4, {frames}), "omt_patchify_ln_u8: frames must be 4-byte aligned");
  OMT_REQUIRE(Cin <= 4, "omt_patchify_ln_u8: Cin=%d must be 1..4", Cin);   // the shared-memory table holds 4 channels
  long long rows;
  int K;
  const int rc = check_gather("omt_patchify_ln_u8", A, A_hi, A_lo, A_rs, ln_w, ln_b, B, Cin, T, H, W, p, pt, first, &rows, &K);
  if (rc != OMT_OK) return rc;
  if (rows == 0) return OMT_OK;
  long long blocks = (rows + PU8_WARPS - 1) / PU8_WARPS;
  if (blocks > (long long)sm_count() * 8) blocks = (long long)sm_count() * 8;   // 8 CTAs of 256 threads fill an SM
  static decltype(&patchify_ln_u8_kernel<2>) const kernels[] = {patchify_ln_u8_kernel<2>, patchify_ln_u8_kernel<6>,
                                                                patchify_ln_u8_kernel<8>};
  OMT_CUDA(launch_k(kernels[gather_nv_index(K)], dim3((unsigned)blocks), dim3(32 * PU8_WARPS), 0, (cudaStream_t)stream,
                    frames, lut, sel, A, A_hi, A_lo, A_rs, ln_w, ln_b, (int)rows, Cin, T, H, W, p, pt, first, eps));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

extern "C" int omt_u8_norm_select(const uint8_t* frames, int B, long long per_sample, int32_t* sel, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(frames && sel, "omt_u8_norm_select: null pointer");
  OMT_REQUIRE(B >= 0 && B <= 65535 && per_sample >= 0, "omt_u8_norm_select: B=%d, per_sample=%lld", B, per_sample);
  if (B == 0) return OMT_OK;
  cudaStream_t st = (cudaStream_t)stream;
  OMT_CUDA(launch_k(u8_sel_init_kernel, dim3((B + 255) / 256), dim3(256), 0, st, sel, B));
  OMT_LAUNCH_CHECK();
  if (per_sample == 0) return OMT_OK;
  long long bx = (per_sample / 16 + 255) / 256;                  // one 16-byte load per thread and block
  const long long cap = ((long long)sm_count() * 8 + B - 1) / B;    // about 8 CTAs per SM over the whole batch
  if (bx > cap) bx = cap;
  if (bx < 1) bx = 1;
  OMT_CUDA(launch_k(u8_sel_scan_kernel, dim3((unsigned)bx, (unsigned)B), dim3(256), 0, st, frames, per_sample, sel));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

// Blocks of 256 threads for the un-patchify grid-stride loops over n items: one per 256 items, at most 32 per SM.
static unsigned unpatchify_blocks(long long n) {
  const long long blocks = (n + 255) / 256, cap = (long long)sm_count() * 32;
  return (unsigned)(blocks < cap ? blocks : cap);
}

extern "C" int omt_unpatchify(const float* P, float* video, int B, int Cin, int T, int H, int W, int p,
                              int pt, int first, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(P && video, "omt_unpatchify: null pointer");
  OMT_REQUIRE(aligned_to(16, {P, video}), "omt_unpatchify: P and video must be 16-byte aligned");
  long long rows;
  int K;
  const int rc = check_patch_geometry("omt_unpatchify", B, Cin, T, H, W, p, pt, first, &rows, &K);
  if (rc != OMT_OK) return rc;
  const long long total4 = rows * (K / 4);
  if (total4 == 0) return OMT_OK;
  OMT_CUDA(launch_k(unpatchify_kernel, dim3(unpatchify_blocks(total4)), dim3(256), 0, (cudaStream_t)stream, P, video, total4,
                    Cin, T, H, W, p, pt, first));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

extern "C" int omt_unpatchify_u8(const float* P, uint8_t* out, int B, int Cin, int T, int H, int W, int p, int pt,
                                 int first, float mul, float add, float lo, float hi, float post, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(P && out, "omt_unpatchify_u8: null pointer");
  OMT_REQUIRE(aligned_to(16, {P}), "omt_unpatchify_u8: P must be 16-byte aligned");
  long long rows;
  int K;
  const int rc = check_patch_geometry("omt_unpatchify_u8", B, Cin, T, H, W, p, pt, first, &rows, &K);
  if (rc != OMT_OK) return rc;
  OMT_REQUIRE(lo >= 0.f && hi * post < 256.f, "omt_unpatchify_u8: clamp range [%g, %g] x %g does not fit a byte", lo, hi, post);
  const long long total = rows * (K / Cin / 4);     // (dt, p1, p2-quad) items
  if (total == 0) return OMT_OK;
  OMT_CUDA(launch_k(unpatchify_u8_kernel, dim3(unpatchify_blocks(total)), dim3(256), 0, (cudaStream_t)stream, P, out, total,
                    Cin, T, H, W, p, pt, first, mul, add, lo, hi, post));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

extern "C" int omt_peg(const float* x, float* y, const float* w27, const float* bias, const int32_t* nbr,
                       int B, int rows_per_b, int C, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(x && y && w27 && bias && nbr, "omt_peg: null pointer");
  OMT_REQUIRE(x != y, "omt_peg: in-place is not supported (stencil)");
  OMT_REQUIRE(aligned_to(16, {x, y, w27, bias}), "omt_peg: x, y, w27 and bias must be 16-byte aligned");
  OMT_REQUIRE(C % 4 == 0 && C / 4 <= 128, "omt_peg: C=%d unsupported (need C %% 4 == 0, C <= 512)", C);
  const long long M = (long long)B * rows_per_b;
  if (M == 0) return OMT_OK;
  static KernelSetup setup;
  const int rc = setup.smem(peg_kernel, 27 * 512 * 4);   // the widest row (C = 512) once
  if (rc != OMT_OK) return rc;
  const size_t smem = (size_t)27 * C * sizeof(float);
  const unsigned blocks = (unsigned)((M + PEG_ROWS - 1) / PEG_ROWS);
  peg_kernel<<<blocks, 128, smem, (cudaStream_t)stream>>>(x, y, w27, bias, nbr, rows_per_b, C, M);
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

// Both PEG entry points: T = every sample's T' (t_off == NULL) or the longest one of a packed batch (t_off = the device table).
// The tile geometry depends on T only, and a CTA whose planes lie past its sample's end exits at once.
static int peg_volume_launch(const char* who, const float* x, float* y, const float* w27, const float* bias,
                             const int32_t* t_off, int B, int T, int h, int w, int C, int temporal, int causal,
                             omt_stream_t stream) {
  OMT_REQUIRE(x && y && w27 && bias, "%s: null pointer", who);
  OMT_REQUIRE(x != y, "%s: in-place is not supported (stencil)", who);
  // both tile kernels gather x in 16-byte chunks and read w27 / bias and write y in channel pairs
  OMT_REQUIRE(aligned_to(16, {x}), "%s: x must be 16-byte aligned", who);
  OMT_REQUIRE(aligned_to(8, {y, w27, bias}), "%s: y, w27 and bias must be 8-byte aligned", who);
  OMT_REQUIRE(C % PEG_CC == 0 && C / PEG_CC <= 65535 && B <= 65535, "%s: C=%d must be a multiple of 16", who, C);
  OMT_REQUIRE(T >= 1 && h >= 1 && w >= 1, "%s: bad volume", who);
  if (B == 0) return OMT_OK;
  // tile geometry: planes per CTA (TT) and rows per CTA (HB) so that threads <= 256 and smem <= ~100 KB
  int RS = (w + 2) * PEG_CC;
  RS += ((16 - RS % 32) + 32) % 32;                  // row stride == 16 (mod 32) floats: 2-way minimum bank pattern
  int TT = T < 5 ? T : 5, HB = 4;
  auto smem_of = [&](int tt, int hb) { return (size_t)(tt + 2) * (hb + 2) * (RS * sizeof(float) + (size_t)(w + 2) * 8); };
  while (HB > 1 && (smem_of(TT, HB) > 112 * 1024 || TT * HB * 8 > 256)) --HB;
  while (TT > 1 && (smem_of(TT, HB) > 112 * 1024 || TT * HB * 8 > 256)) --TT;
  const size_t smem = smem_of(TT, HB);
  OMT_REQUIRE(smem <= 200 * 1024, "%s: row of %d tokens does not fit the shared-memory tile", who, w);
  static KernelSetup setup3, setup4;
  int rc = setup3.smem(peg_tile_kernel, smem);
  if (rc != OMT_OK) return rc;
  const int threads = ((TT * HB * 8 + 31) / 32) * 32;
  dim3 grid(((T + TT - 1) / TT) * ((h + HB - 1) / HB), C / PEG_CC, B);
  const bool fast_ok = T <= 64 && w <= 254;
  const bool v4 = g_peg_kernel == 4 && fast_ok;
  if (v4) {
    // planes of a tile that lie inside the volume (the others are one shared zero row): the maximum over the t-blocks
    const int pad_lo = causal ? 2 : 1;
    int vp = 1;
    for (int t0 = 0; t0 < T; t0 += TT) {
      const int lo = t0 - pad_lo < 0 ? 0 : t0 - pad_lo, hi = t0 - pad_lo + TT + 2 > T ? T : t0 - pad_lo + TT + 2;
      if (hi - lo > vp) vp = hi - lo;
    }
    const int zrow = vp * (HB + 2);
    const size_t smem4 = (size_t)(zrow + 1) * RS * sizeof(float);
    if ((rc = setup4.smem(peg_tile4_kernel, smem4)) != OMT_OK) return rc;
    OMT_CUDA(launch_k(peg_tile4_kernel, grid, dim3(threads), smem4, (cudaStream_t)stream, x, y, w27, bias, T, h, w, C, temporal, causal, TT, HB, RS, zrow, t_off));
  } else {
    OMT_CUDA(launch_k(peg_tile_kernel, grid, dim3(threads), smem, (cudaStream_t)stream, x, y, w27, bias, T, h, w, C, temporal, causal, TT, HB, RS, t_off));
  }
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

extern "C" int omt_peg_volume(const float* x, float* y, const float* w27, const float* bias, int B, int T, int h,
                              int w, int C, int temporal, int causal, omt_stream_t stream) {
  OMT_ENTER();
  return peg_volume_launch("omt_peg_volume", x, y, w27, bias, nullptr, B, T, h, w, C, temporal, causal, stream);
}

extern "C" int omt_peg_volume_varlen(const float* x, float* y, const float* w27, const float* bias, const int32_t* t_off_host,
                                     const int32_t* t_off, int B, int M, int h, int w, int C, int temporal, int causal,
                                     omt_stream_t stream) {
  OMT_ENTER();
  int t_max = 0;
  const int rc = check_t_off("omt_peg_volume_varlen", t_off_host, t_off, B, M, (long long)h * w, &t_max);
  if (rc) return rc;
  return peg_volume_launch("omt_peg_volume_varlen", x, y, w27, bias, t_off, B, t_max < 1 ? 1 : t_max, h, w, C, temporal,
                           causal, stream);
}

extern "C" int omt_qk_prep(float* q, int ldq, float* k, int ldk, const float* q_scale, const float* k_scale,
                           const float* rope_cos, const float* rope_sin, int M, int N, int heads,
                           omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(q && k && q_scale && k_scale, "omt_qk_prep: null pointer");
  OMT_REQUIRE((rope_cos == nullptr) == (rope_sin == nullptr), "omt_qk_prep: cos/sin must both be given");
  OMT_REQUIRE(ldq % 2 == 0 && ldk % 2 == 0 && N > 0, "omt_qk_prep: bad leading dims");
  OMT_REQUIRE(aligned_to(8, {q, k, q_scale, k_scale}), "omt_qk_prep: q, k, q_scale and k_scale must be 8-byte aligned");
  if (M == 0) return OMT_OK;
  OMT_CUDA(launch_k(qk_prep_kernel, dim3((M + 7) / 8), dim3(256), 0, (cudaStream_t)stream, q, ldq, k, ldk, q_scale, k_scale,
                    rope_cos, rope_sin, M, N, heads));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}
