// omt_resample_u8: Pillow's 8-bit resize (libImaging/Resample.c, ImagingResampleHorizontal_8bpc / _Vertical_8bpc) of a
// ragged batch of uint8 RGB images, with the loaders' random crop and horizontal flip as output index maps.
//
// Pillow resizes in two int32 passes over 22-bit fixed-point coefficients: horizontal (source rows -> an 8-bit
// intermediate image, clip8 per byte), then vertical.  The coefficients are computed on the host in float64 exactly as
// precompute_coeffs + normalize_coeffs_8bpc do (layout.resample_coeffs); this kernel only does the integer arithmetic,
// so its bytes are Pillow's.  Each CTA owns an RS_TW x RS_TH output tile of one image: the horizontal pass covers only the
// source rows the tile's vertical taps reach and lands in shared memory as clip8'ed bytes (Pillow's intermediate image),
// in chunks of RS_CHUNK rows, so any tap count (5 for a bicubic upscale, 65 for a 16x downscale, hundreds beyond) fits.
// Integer sums are exact, so splitting a column's vertical taps across chunks changes nothing.  Pillow's Image.resize
// runs the vertical pass first for images taller than 100x their width (v_first); those few go byte by byte.
#include "omt_common.cuh"
#include <limits.h>

using namespace omt;

namespace {

constexpr int RS_TW = 64;        // output columns per tile (one per thread of a row group)
constexpr int RS_TH = 16;        // output rows per tile
constexpr int RS_THREADS = 256;  // 4 row groups of 64 threads
constexpr int RS_GROUPS = RS_THREADS / RS_TW;
constexpr int RS_CHUNK = 128;    // intermediate rows in shared memory at a time: 128 x 64 x 3 B = 24 KB
constexpr int RS_PREC = 22;      // Resample.c PRECISION_BITS (32 - 8 - 2)

__device__ __forceinline__ int clip8(int v) {   // Resample.c clip8
  return v >= (1 << RS_PREC << 8) ? 255 : (v <= 0 ? 0 : (v >> RS_PREC));
}

__global__ void __launch_bounds__(RS_THREADS)
resample_u8_kernel(const uint8_t* __restrict__ src, const omt_resample_desc* __restrict__ desc,
                   const int32_t* __restrict__ tab, uint8_t* __restrict__ out, int oh, int ow) {
  __shared__ uint8_t inter[RS_CHUNK][RS_TW * 3];
  pdl_sync();
  const omt_resample_desc d = desc[blockIdx.z];
  const int ox0 = blockIdx.x * RS_TW, oy0 = blockIdx.y * RS_TH;
  const int th = min(RS_TH, oh - oy0);
  const int lc = threadIdx.x % RS_TW, rg = threadIdx.x / RS_TW;
  const int ox = ox0 + lc;
  const bool col_ok = ox < ow;
  const uint8_t* img = src + d.src;

  // source rows [ys, ye) the tile's vertical taps reach (the crop shifts rows; a flip only mirrors columns)
  int ys = INT_MAX, ye = 0;
  for (int i = 0; i < th; ++i) {
    const int ry = d.y0 + oy0 + i;
    const int a = d.need_v ? __ldg(tab + d.vb + 2 * ry) : ry;
    const int n = d.need_v ? __ldg(tab + d.vb + 2 * ry + 1) : 1;
    ys = min(ys, a);
    ye = max(ye, a + n);
  }

  // this thread's column of the resized image and its horizontal taps
  const int rx = d.flip ? d.x0 + (ow - 1 - ox) : d.x0 + ox;
  int hx = rx, hn = 1;
  const int32_t* hk = nullptr;
  if (col_ok && d.need_h) {
    hx = __ldg(tab + d.hb + 2 * rx);
    hn = __ldg(tab + d.hb + 2 * rx + 1);
    hk = tab + d.hc + (long long)rx * d.hk;
  }

  constexpr int RPT = RS_TH / RS_GROUPS;
  if (d.v_first) {   // tall images (H > 100 W): vertical, clip8, then horizontal, per output byte straight from the source
    if (!col_ok) return;
    for (int j = 0; j < RPT; ++j) {
      const int i = rg + j * RS_GROUPS;
      if (i >= th) break;
      const int ry = d.y0 + oy0 + i;
      const int a = __ldg(tab + d.vb + 2 * ry), n = __ldg(tab + d.vb + 2 * ry + 1);
      const int32_t* vk = tab + d.vc + (long long)ry * d.vk;
      int s[3] = {1 << (RS_PREC - 1), 1 << (RS_PREC - 1), 1 << (RS_PREC - 1)};
      for (int x = 0; x < hn; ++x) {
        const uint8_t* p = img + ((long long)a * d.W + hx + x) * 3;
        int v[3] = {1 << (RS_PREC - 1), 1 << (RS_PREC - 1), 1 << (RS_PREC - 1)};
        for (int y = 0; y < n; ++y, p += (long long)d.W * 3) {
          const int k = __ldg(vk + y);
#pragma unroll
          for (int c = 0; c < 3; ++c) v[c] += __ldg(p + c) * k;
        }
        const int k = __ldg(hk + x);
#pragma unroll
        for (int c = 0; c < 3; ++c) s[c] += clip8(v[c]) * k;
      }
      uint8_t* o = out + (((long long)blockIdx.z * oh + oy0 + i) * ow + ox) * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) o[c] = (uint8_t)clip8(s[c]);
    }
    return;
  }

  // rows rg, rg + 4, ... of the tile: vertical accumulators (or, without a vertical pass, the copied bytes)
  int acc[RPT][3];
#pragma unroll
  for (int j = 0; j < RPT; ++j) acc[j][0] = acc[j][1] = acc[j][2] = d.need_v ? 1 << (RS_PREC - 1) : 0;

  for (int c0 = ys; c0 < ye; c0 += RS_CHUNK) {
    const int c1 = min(ye, c0 + RS_CHUNK);
    __syncthreads();                                   // the previous chunk has been read
    if (col_ok) {
      for (int r = c0 + rg; r < c1; r += RS_GROUPS) {
        const uint8_t* row = img + (long long)r * d.W * 3;
        uint8_t* o = &inter[r - c0][lc * 3];
        if (d.need_h) {
          int s0 = 1 << (RS_PREC - 1), s1 = s0, s2 = s0;
          const uint8_t* p = row + hx * 3;
          for (int x = 0; x < hn; ++x, p += 3) {
            const int k = __ldg(hk + x);
            s0 += __ldg(p) * k;
            s1 += __ldg(p + 1) * k;
            s2 += __ldg(p + 2) * k;
          }
          o[0] = (uint8_t)clip8(s0);
          o[1] = (uint8_t)clip8(s1);
          o[2] = (uint8_t)clip8(s2);
        } else {
          o[0] = __ldg(row + rx * 3);
          o[1] = __ldg(row + rx * 3 + 1);
          o[2] = __ldg(row + rx * 3 + 2);
        }
      }
    }
    __syncthreads();
    if (col_ok) {
#pragma unroll
      for (int j = 0; j < RPT; ++j) {
        const int i = rg + j * RS_GROUPS;
        if (i >= th) continue;
        const int ry = d.y0 + oy0 + i;
        if (d.need_v) {
          const int a = __ldg(tab + d.vb + 2 * ry), n = __ldg(tab + d.vb + 2 * ry + 1);
          const int32_t* vk = tab + d.vc + (long long)ry * d.vk;
          const int y1 = min(a + n, c1);
          for (int y = max(a, c0); y < y1; ++y) {
            const int k = __ldg(vk + (y - a));
            const uint8_t* p = &inter[y - c0][lc * 3];
            acc[j][0] += p[0] * k;
            acc[j][1] += p[1] * k;
            acc[j][2] += p[2] * k;
          }
        } else if (ry >= c0 && ry < c1) {
          const uint8_t* p = &inter[ry - c0][lc * 3];
          acc[j][0] = p[0];
          acc[j][1] = p[1];
          acc[j][2] = p[2];
        }
      }
    }
  }

  if (!col_ok) return;
#pragma unroll
  for (int j = 0; j < RPT; ++j) {
    const int i = rg + j * RS_GROUPS;
    if (i >= th) continue;
    uint8_t* o = out + (((long long)blockIdx.z * oh + oy0 + i) * ow + ox) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = (uint8_t)(d.need_v ? clip8(acc[j][c]) : acc[j][c]);
  }
}

// omt_resample_clips: the Latte video loaders' ToTensorVideo -> flip -> bilinear F.interpolate (+ centre crop) ->
// Normalize, in torch's fp32 CPU arithmetic (either of its two bilinear kernels, per clip: desc.form).  Its own kernel:
// nothing here is shared with Pillow's integer resize.
// Each CTA owns RC_TW output columns (one per thread) x RC_TH rows of one frame of one clip; a thread's horizontal table
// entry is loaded once, and each output row reads exactly two source rows.  Stores run along w within a channel plane.
// OUT = OUT_FVD (omt_fvd_preprocess): fvd.py's preprocess instead of the loaders' Normalize.  The byte table holds the
// value each byte stands for (table sel[b] of two when sel is given), the result is 2 y / 255 - 1 in that order, and a
// frame leaves channels-last as [oh][ow][4] with channel 3 zero (the I3D input layout).
// OUT = OUT_FID (omt_fid_preprocess): pytorch-fid's ToTensor -> F.interpolate -> 2 x - 1.  The same layout and tables, but
// the byte table already holds byte / 255 (the division comes before the resize), and the result is 2 y - 1.
constexpr int RC_TW = 128;
constexpr int RC_TH = 8;
enum { OUT_NORMALIZE = 0, OUT_FVD = 1, OUT_FID = 2 };

template <int OUT>
__device__ __forceinline__ void resample_clips_body(const uint8_t* __restrict__ src, const omt_clip_desc* __restrict__ desc,
                                                    const int4* __restrict__ tab, const float* __restrict__ norm,
                                                    float* __restrict__ out, int F, int oh, int ow,
                                                    const int32_t* __restrict__ sel) {
  constexpr bool FVD = OUT != OUT_NORMALIZE;     // a feature network's input: byte table sel[b], [oh][ow][4] out
  __shared__ float lut[256];
  pdl_sync();
  const int b = blockIdx.z / F, f = blockIdx.z % F;
  const omt_clip_desc d = desc[b];
  if constexpr (FVD) {
    if (sel != nullptr) norm += 256 * __ldg(sel + b);
  }
  for (int i = threadIdx.x; i < 256; i += RC_TW) lut[i] = __ldg(norm + i);
  __syncthreads();
  const int ox = blockIdx.x * RC_TW + threadIdx.x;
  if (ox >= ow) return;
  float mean[3], stdv[3];
  if constexpr (!FVD) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      mean[c] = __ldg(norm + 256 + c);
      stdv[c] = __ldg(norm + 259 + c);
    }
  }
  const int4 ew = __ldg(tab + d.th / 4 + d.cx + ox);
  const int x0 = d.flip ? d.W - 1 - (d.x0 + ew.x) : d.x0 + ew.x;   // the flip comes before the resize: mirror the source
  const int x1 = d.flip ? d.W - 1 - (d.x0 + ew.y) : d.x0 + ew.y;
  const float l0w = __int_as_float(ew.z), l1w = __int_as_float(ew.w);
  const uint8_t* frame = src + d.src + (long long)f * d.H * d.W * 3;
  const long long plane = (long long)oh * ow;
  float* o = out + ((long long)b * 3 * F + f) * plane + ox;        // channel c at + c * F * plane
  const int y_end = min(oh, (int)blockIdx.y * RC_TH + RC_TH);
  for (int oy = blockIdx.y * RC_TH; oy < y_end; ++oy) {
    const int4 eh = __ldg(tab + d.tv / 4 + d.cy + oy);
    const float l0h = __int_as_float(eh.z), l1h = __int_as_float(eh.w);
    const uint8_t* r0 = frame + (long long)(d.y0 + eh.x) * d.W * 3;
    const uint8_t* r1 = frame + (long long)(d.y0 + eh.y) * d.W * 3;
    // torch's CPU kernels: each fma rounds once; the products and the division are never contracted or reassociated
    const float w00 = __fmul_rn(l0h, l0w), w01 = __fmul_rn(l0h, l1w), w10 = __fmul_rn(l1h, l0w), w11 = __fmul_rn(l1h, l1w);
    float y[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float x00 = lut[__ldg(r0 + x0 * 3 + c)], x01 = lut[__ldg(r0 + x1 * 3 + c)];
      const float x10 = lut[__ldg(r1 + x0 * 3 + c)], x11 = lut[__ldg(r1 + x1 * 3 + c)];
      float v;
      if (d.form) {
        v = __fmaf_rn(x11, w11, __fmaf_rn(x10, w10, __fmaf_rn(x00, w00, __fmul_rn(x01, w01))));
      } else {
        const float t0 = __fmaf_rn(x00, l0w, __fmul_rn(x01, l1w));
        const float t1 = __fmaf_rn(x10, l0w, __fmul_rn(x11, l1w));
        v = __fmaf_rn(t0, l0h, __fmul_rn(t1, l1h));
      }
      if constexpr (OUT == OUT_FID) y[c] = __fsub_rn(__fmul_rn(2.f, v), 1.f);
      else if constexpr (FVD) y[c] = __fsub_rn(__fdiv_rn(__fmul_rn(2.f, v), 255.f), 1.f);
      else o[c * F * plane + (long long)oy * ow] = __fdiv_rn(__fsub_rn(v, mean[c]), stdv[c]);
    }
    if constexpr (FVD)
      reinterpret_cast<float4*>(out)[((long long)blockIdx.z * oh + oy) * ow + ox] = make_float4(y[0], y[1], y[2], 0.f);
  }
}

__global__ void __launch_bounds__(RC_TW)
resample_clips_kernel(const uint8_t* __restrict__ src, const omt_clip_desc* __restrict__ desc,
                      const int4* __restrict__ tab, const float* __restrict__ norm, float* __restrict__ out, int F,
                      int oh, int ow) {
  resample_clips_body<OUT_NORMALIZE>(src, desc, tab, norm, out, F, oh, ow, nullptr);
}

__global__ void __launch_bounds__(RC_TW)
fvd_preprocess_kernel(const uint8_t* __restrict__ src, const omt_clip_desc* __restrict__ desc,
                      const int4* __restrict__ tab, const float* __restrict__ lut, const int32_t* __restrict__ sel,
                      float* __restrict__ out, int F, int oh, int ow) {
  resample_clips_body<OUT_FVD>(src, desc, tab, lut, out, F, oh, ow, sel);
}

__global__ void __launch_bounds__(RC_TW)
fid_preprocess_kernel(const uint8_t* __restrict__ src, const omt_clip_desc* __restrict__ desc,
                      const int4* __restrict__ tab, const float* __restrict__ lut, const int32_t* __restrict__ sel,
                      float* __restrict__ out, int oh, int ow) {
  resample_clips_body<OUT_FID>(src, desc, tab, lut, out, 1, oh, ow, sel);
}

// One axis table of a clip: [n_out][4] entries at word `off` inside the table, every (i0, i1) inside an axis of n_in.
bool clip_axis_ok(const int32_t* tab_host, long long tab_len, int off, int n_out, int n_in) {
  if (off < 0 || off % 4 != 0 || off + 4LL * n_out > tab_len) return false;
  for (int i = 0; i < n_out; ++i) {
    const int i0 = tab_host[off + 4 * i], i1 = tab_host[off + 4 * i + 1];
    if (i0 < 0 || i1 < i0 || i1 >= n_in) return false;
  }
  return true;
}

// One axis of a descriptor: its (xmin, n) bounds [out][2] at `b` and coefficients [out][k] at `c` lie inside the table,
// and every output index's taps lie inside the source axis of length `in`.
bool axis_ok(const int32_t* tab_host, long long tab_len, int b, int c, int k, int out, int in) {
  if (b < 0 || c < 0 || k < 1 || b + 2LL * out > tab_len || c + (long long)out * k > tab_len) return false;
  for (int i = 0; i < out; ++i) {
    const int xmin = tab_host[b + 2 * i], n = tab_host[b + 2 * i + 1];
    if (xmin < 0 || n < 0 || n > k || (long long)xmin + n > in) return false;
  }
  return true;
}

}  // namespace

extern "C" int omt_resample_u8(const uint8_t* src, long long src_bytes, const omt_resample_desc* desc,
                               const omt_resample_desc* desc_host, const int32_t* tab, const int32_t* tab_host,
                               long long tab_len, int B, int oh, int ow, uint8_t* out, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(src && desc && desc_host && out && ((tab == nullptr) == (tab_host == nullptr)) && ((tab == nullptr) == (tab_len == 0)),
              "omt_resample_u8: null pointer");
  OMT_REQUIRE(B >= 1 && B <= 65535 && oh >= 1 && ow >= 1 && src_bytes >= 0 && tab_len >= 0,
              "omt_resample_u8: B=%d, output %dx%d, src_bytes=%lld, tab_len=%lld", B, oh, ow, src_bytes, tab_len);
  OMT_REQUIRE((uintptr_t)desc % 8 == 0 && (uintptr_t)tab % 4 == 0, "omt_resample_u8: desc must be 8-byte and tab 4-byte aligned");
  for (int b = 0; b < B; ++b) {
    const omt_resample_desc& d = desc_host[b];
    OMT_REQUIRE(d.H >= 1 && d.W >= 1 && d.rh >= 1 && d.rw >= 1,
                "omt_resample_u8: image %d: source %dx%d, resized %dx%d", b, d.H, d.W, d.rh, d.rw);
    OMT_REQUIRE(d.src >= 0 && d.src + (long long)d.H * d.W * 3 <= src_bytes,
                "omt_resample_u8: image %d: bytes [%lld, +%lld) outside the %lld source bytes", b, d.src,
                (long long)d.H * d.W * 3, src_bytes);
    OMT_REQUIRE(d.y0 >= 0 && d.x0 >= 0 && (long long)d.y0 + oh <= d.rh && (long long)d.x0 + ow <= d.rw,
                "omt_resample_u8: image %d: crop %dx%d at (%d, %d) outside the resized %dx%d image", b, oh, ow, d.y0,
                d.x0, d.rh, d.rw);
    OMT_REQUIRE((d.flip | d.need_h | d.need_v | d.v_first) >= 0 && (d.flip | d.need_h | d.need_v | d.v_first) <= 1,
                "omt_resample_u8: image %d: flip / need_h / need_v / v_first must be 0 or 1", b);
    OMT_REQUIRE(!d.v_first || (d.need_h && d.need_v), "omt_resample_u8: image %d: v_first without both passes", b);
    OMT_REQUIRE(d.need_h || d.rw == d.W, "omt_resample_u8: image %d: no horizontal pass but width %d -> %d", b, d.W, d.rw);
    OMT_REQUIRE(d.need_v || d.rh == d.H, "omt_resample_u8: image %d: no vertical pass but height %d -> %d", b, d.H, d.rh);
    OMT_REQUIRE(!d.need_h || axis_ok(tab_host, tab_len, d.hb, d.hc, d.hk, d.rw, d.W),
                "omt_resample_u8: image %d: horizontal table outside the table or taps outside the source", b);
    OMT_REQUIRE(!d.need_v || axis_ok(tab_host, tab_len, d.vb, d.vc, d.vk, d.rh, d.H),
                "omt_resample_u8: image %d: vertical table outside the table or taps outside the source", b);
  }
  dim3 grid((ow + RS_TW - 1) / RS_TW, (oh + RS_TH - 1) / RS_TH, B);
  OMT_CUDA(launch_k(resample_u8_kernel, grid, dim3(RS_THREADS), 0, (cudaStream_t)stream, src, desc, tab, out, oh, ow));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

// The checks both clip entry points make before their launch (`who` names the entry point in the message).
static int check_clips(const char* who, const uint8_t* src, long long src_bytes, const omt_clip_desc* desc,
                       const omt_clip_desc* desc_host, const int32_t* tab, const int32_t* tab_host, long long tab_len,
                       const float* norm, int B, int F, int oh, int ow, float* out) {
  OMT_REQUIRE(src && desc && desc_host && tab && tab_host && norm && out, "%s: null pointer", who);
  OMT_REQUIRE(B >= 1 && F >= 1 && (long long)B * F <= 65535 && oh >= 1 && ow >= 1 && src_bytes >= 0 && tab_len >= 0,
              "%s: B=%d, F=%d, output %dx%d, src_bytes=%lld, tab_len=%lld", who, B, F, oh, ow, src_bytes, tab_len);
  for (int b = 0; b < B; ++b) {
    const omt_clip_desc& d = desc_host[b];
    OMT_REQUIRE(d.H >= 1 && d.W >= 1 && d.wh >= 1 && d.ww >= 1 && d.rh >= 1 && d.rw >= 1,
                "%s: clip %d: source %dx%d, window %dx%d, resized %dx%d", who, b, d.H, d.W, d.wh, d.ww, d.rh, d.rw);
    OMT_REQUIRE(d.src >= 0 && d.src + (long long)F * d.H * d.W * 3 <= src_bytes,
                "%s: clip %d: bytes [%lld, +%lld) outside the %lld source bytes", who, b, d.src,
                (long long)F * d.H * d.W * 3, src_bytes);
    OMT_REQUIRE(d.y0 >= 0 && d.x0 >= 0 && (long long)d.y0 + d.wh <= d.H && (long long)d.x0 + d.ww <= d.W,
                "%s: clip %d: window %dx%d at (%d, %d) outside the %dx%d frame", who, b, d.wh, d.ww, d.y0, d.x0, d.H, d.W);
    OMT_REQUIRE(d.cy >= 0 && d.cx >= 0 && (long long)d.cy + oh <= d.rh && (long long)d.cx + ow <= d.rw,
                "%s: clip %d: crop %dx%d at (%d, %d) outside the resized %dx%d frame", who, b, oh, ow, d.cy, d.cx, d.rh,
                d.rw);
    OMT_REQUIRE((d.flip | d.form) >= 0 && (d.flip | d.form) <= 1, "%s: clip %d: flip / form must be 0 or 1", who, b);
    OMT_REQUIRE(clip_axis_ok(tab_host, tab_len, d.tv, d.rh, d.wh),
                "%s: clip %d: vertical table outside the table or indices outside the window", who, b);
    OMT_REQUIRE(clip_axis_ok(tab_host, tab_len, d.th, d.rw, d.ww),
                "%s: clip %d: horizontal table outside the table or indices outside the window", who, b);
  }
  return OMT_OK;
}

extern "C" int omt_resample_clips(const uint8_t* src, long long src_bytes, const omt_clip_desc* desc,
                                  const omt_clip_desc* desc_host, const int32_t* tab, const int32_t* tab_host,
                                  long long tab_len, const float* norm, int B, int F, int oh, int ow, float* out,
                                  omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(aligned_to(8, {desc}) && aligned_to(16, {tab}) && aligned_to(4, {norm, out}),
              "omt_resample_clips: desc must be 8-byte, tab 16-byte and norm / out 4-byte aligned");
  int rc = check_clips("omt_resample_clips", src, src_bytes, desc, desc_host, tab, tab_host, tab_len, norm, B, F, oh, ow, out);
  if (rc != OMT_OK) return rc;
  dim3 grid((ow + RC_TW - 1) / RC_TW, (oh + RC_TH - 1) / RC_TH, B * F);
  OMT_CUDA(launch_k(resample_clips_kernel, grid, dim3(RC_TW), 0, (cudaStream_t)stream, src, desc,
                    reinterpret_cast<const int4*>(tab), norm, out, F, oh, ow));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

extern "C" int omt_fvd_preprocess(const uint8_t* src, long long src_bytes, const omt_clip_desc* desc,
                                  const omt_clip_desc* desc_host, const int32_t* tab, const int32_t* tab_host,
                                  long long tab_len, const float* lut, const int32_t* sel, int B, int F, int oh,
                                  int ow, float* out, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(aligned_to(4, {sel}), "omt_fvd_preprocess: sel must be 4-byte aligned");
  OMT_REQUIRE(aligned_to(8, {desc}) && aligned_to(16, {tab, out}) && aligned_to(4, {lut}),
              "omt_fvd_preprocess: desc must be 8-byte, tab / out 16-byte and lut 4-byte aligned");
  int rc = check_clips("omt_fvd_preprocess", src, src_bytes, desc, desc_host, tab, tab_host, tab_len, lut, B, F, oh, ow, out);
  if (rc != OMT_OK) return rc;
  dim3 grid((ow + RC_TW - 1) / RC_TW, (oh + RC_TH - 1) / RC_TH, B * F);
  OMT_CUDA(launch_k(fvd_preprocess_kernel, grid, dim3(RC_TW), 0, (cudaStream_t)stream, src, desc,
                    reinterpret_cast<const int4*>(tab), lut, sel, out, F, oh, ow));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

extern "C" int omt_fid_preprocess(const uint8_t* src, long long src_bytes, const omt_clip_desc* desc,
                                  const omt_clip_desc* desc_host, const int32_t* tab, const int32_t* tab_host,
                                  long long tab_len, const float* lut, const int32_t* sel, int B, int oh, int ow,
                                  float* out, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(aligned_to(4, {sel}), "omt_fid_preprocess: sel must be 4-byte aligned");
  OMT_REQUIRE(aligned_to(8, {desc}) && aligned_to(16, {tab, out}) && aligned_to(4, {lut}),
              "omt_fid_preprocess: desc must be 8-byte, tab / out 16-byte and lut 4-byte aligned");
  int rc = check_clips("omt_fid_preprocess", src, src_bytes, desc, desc_host, tab, tab_host, tab_len, lut, B, 1, oh, ow, out);
  if (rc != OMT_OK) return rc;
  dim3 grid((ow + RC_TW - 1) / RC_TW, (oh + RC_TH - 1) / RC_TH, B);
  OMT_CUDA(launch_k(fid_preprocess_kernel, grid, dim3(RC_TW), 0, (cudaStream_t)stream, src, desc,
                    reinterpret_cast<const int4*>(tab), lut, sel, out, oh, ow));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}
