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

// The bilinear clip kernel of omt_resample_clips, omt_fvd_preprocess, omt_fid_preprocess, omt_fvd_suite_preprocess,
// omt_is_preprocess and omt_eval_downsample: torch's fp32 CPU F.interpolate(bilinear, align_corners=False) of B clips
// of F frames, bit for bit, in either of its two kernels per clip (desc.form).  Nothing here is shared with Pillow's
// integer resize above.  A source policy says what one sample of a frame is worth in fp32; an output policy says what
// the three resized channel values of a pixel become and where they go.  Each policy keeps the exact intrinsics of the
// reference it stands for.
// Each CTA owns RC_TW output columns (one per thread) x RC_TH rows of one frame of one clip (blockIdx.z = b F + f); a
// thread's horizontal table entry is loaded once, and each output row reads exactly two source rows.  The window origin
// and the flip apply to every entry point; the host check of those that have neither refuses them.
constexpr int RC_TW = 128;
constexpr int RC_TH = 8;

// Source policies.  begin() runs once per thread before any thread leaves (a byte table is loaded there) and points
// the policy at frame f of clip b; then (y, x, c) is channel c of the frame's sample at row y0 + y, column x, as fp32.
// begin() adds the window's y0 once: added in the row loop, it cost the table instances 8 registers.
// lut[byte] of (F, H, W, 3) bytes through a 256-entry table in shared memory, table sel[b] of two when sel is given:
// the loaders (to_tensor's byte / 255), FVD (float(byte) or a byte map), FID (byte / 255) and the eval downsample's
// real clips (VideoNorm(byte) + 0.5).
struct ByteTable {
  static constexpr bool TABLE = true;
  const uint8_t* src;
  const float* lut;
  const int32_t* sel;
  const float* t = nullptr;
  const uint8_t* frame = nullptr;
  int W = 0;
  __device__ void begin(const omt_clip_desc& d, int b, int f, int) {
    __shared__ float s[256];
    const float* g = sel != nullptr ? lut + 256 * __ldg(sel + b) : lut;
    for (int i = threadIdx.x; i < 256; i += RC_TW) s[i] = __ldg(g + i);
    __syncthreads();
    t = s;
    frame = src + d.src + ((long long)f * d.H + d.y0) * d.W * 3;
    W = d.W;
  }
  __device__ float operator()(int y, int x, int c) const { return t[__ldg(frame + (long long)y * W * 3 + x * 3 + c)]; }
};

// The video-metric suite's and the Inception Score's frames (desc.src counts elements; the frames of a clip follow each
// other, so a clip stored with a longer time axis is read as its first F frames):
//   OMT_FVDS_U8:        (F, H, W, 3) bytes, (float)byte / 255, a true division;
//   OMT_FVDS_F32:       fp32 (F, C, H, W), C == 1 read by every channel, used as they are (styleganv);
//   OMT_FVDS_F32_TRUNC: the same through videogpt's (videos * 255).numpy().astype(np.uint8), then .float() / 255.  The
//                       cast truncates to int32 and keeps the low byte, as the x86-64 conversion does for products
//                       inside the int32 range.
__device__ __forceinline__ float suite_u8_value(int b) { return __fdiv_rn((float)b, 255.f); }

template <int FORM>
struct SuiteFrames {
  static constexpr bool TABLE = false;
  const void* src;
  int C;
  long long frame = 0;
  int H = 0, W = 0;
  __device__ void begin(const omt_clip_desc& d, int, int f, int) {
    frame = d.src + (FORM == OMT_FVDS_U8 ? 3 * ((long long)f * d.H + d.y0) : (long long)f * C * d.H + d.y0) * d.W;
    H = d.H;
    W = d.W;
  }
  __device__ float operator()(int y, int x, int c) const {
    if constexpr (FORM == OMT_FVDS_U8) {
      return suite_u8_value(__ldg(static_cast<const uint8_t*>(src) + frame + ((long long)y * W + x) * 3 + c));
    } else {
      const float v = __ldg(static_cast<const float*>(src) + frame + ((long long)(C == 1 ? 0 : c) * H + y) * W + x);
      if constexpr (FORM == OMT_FVDS_F32) return v;
      return suite_u8_value(__float2int_rz(__fmul_rn(v, 255.f)) & 255);
    }
  }
};

// clamp(x + 0.5, 0, 1) of the decoder's fp32 reconstruction, (3, F, H, W) per clip: the eval downsample's other side.
struct ClampedPlanes {
  static constexpr bool TABLE = false;
  const float* src;
  const float* frame = nullptr;
  long long cstride = 0;
  int W = 0;
  __device__ void begin(const omt_clip_desc& d, int, int f, int F) {
    const long long plane = (long long)d.H * d.W;
    frame = src + d.src + f * plane + (long long)d.y0 * d.W;
    cstride = F * plane;
    W = d.W;
  }
  __device__ float operator()(int y, int x, int c) const {
    const float v = __fadd_rn(__ldg(frame + c * cstride + (long long)y * W + x), 0.5f);
    return v != v ? v : fminf(fmaxf(v, 0.f), 1.f);        // torch.clamp keeps a NaN
  }
};

// Output policies: (y, b, f, F, oy, ox, oh, ow) writes the resized values y[3] of output pixel (oy, ox) of frame f of
// clip b.  Each pointer `out` is aligned to the size of what it points to.
// The loaders' Normalize, (y - mean_c) / std_c with a true division, channel-planar (B, 3, F, oh, ow); norm is the
// loaders' table: 256 byte values, then mean[3], then std[3].
struct NormalizePlanes {
  float* out;
  const float* norm;
  __device__ void operator()(const float (&y)[3], int b, int f, int F, int oy, int ox, int oh, int ow) const {
    const long long plane = (long long)oh * ow;
    float* o = out + ((long long)b * 3 * F + f) * plane + (long long)oy * ow + ox;
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c * F * plane] = __fdiv_rn(__fsub_rn(y[c], __ldg(norm + 256 + c)), __ldg(norm + 259 + c));
  }
};

// A feature network's input, channels-last (B, F, oh, ow, 4) with channel 3 zero, one 16-byte store per pixel, after
// fvd.py's 2 y / 255 - 1 (in that order), pytorch-fid's 2 y - 1, the suite's (y - 0.5) * 2, or the Inception Score's
// y as it is.
enum { AFF_FVD, AFF_FID, AFF_SUITE, AFF_NONE };
template <int AFF>
struct Float4Pixels {
  float4* out;
  __device__ static float affine(float v) {
    if constexpr (AFF == AFF_FVD) return __fsub_rn(__fdiv_rn(__fmul_rn(2.f, v), 255.f), 1.f);
    else if constexpr (AFF == AFF_FID) return __fsub_rn(__fmul_rn(2.f, v), 1.f);
    else if constexpr (AFF == AFF_SUITE) return __fmul_rn(__fsub_rn(v, 0.5f), 2.f);
    else return v;
  }
  __device__ void operator()(const float (&y)[3], int, int, int, int oy, int ox, int oh, int ow) const {
    out[((long long)blockIdx.z * oh + oy) * ow + ox] = make_float4(affine(y[0]), affine(y[1]), affine(y[2]), 0.f);
  }
};

// The eval downsample's * 255 and .byte(): the product truncated to int32 and its low byte kept, as on x86-64, written
// channels-last as (B, F, oh, ow, 3) uint8.
struct BytePixels {
  uint8_t* out;
  __device__ void operator()(const float (&y)[3], int, int, int, int oy, int ox, int oh, int ow) const {
    uint8_t* o = out + (((long long)blockIdx.z * oh + oy) * ow + ox) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = (uint8_t)(__float2int_rz(__fmul_rn(y[c], 255.f)) & 255);
  }
};

template <class Src, class Out>
__global__ void __launch_bounds__(RC_TW)
bilinear_clips_kernel(Src src, const Out out, const omt_clip_desc* __restrict__ desc, const int4* __restrict__ tab,
                      int F, int oh, int ow) {
  pdl_sync();
  const int b = blockIdx.z / F, f = blockIdx.z % F;
  const omt_clip_desc d = desc[b];
  src.begin(d, b, f, F);
  const int ox = blockIdx.x * RC_TW + threadIdx.x;
  if (ox >= ow) return;
  const int4 ew = __ldg(tab + d.th / 4 + d.cx + ox);
  const int x0 = d.flip ? d.W - 1 - (d.x0 + ew.x) : d.x0 + ew.x;   // the flip comes before the resize: mirror the source
  const int x1 = d.flip ? d.W - 1 - (d.x0 + ew.y) : d.x0 + ew.y;
  const float l0w = __int_as_float(ew.z), l1w = __int_as_float(ew.w);
  const int y_end = min(oh, (int)blockIdx.y * RC_TH + RC_TH);
  for (int oy = blockIdx.y * RC_TH; oy < y_end; ++oy) {
    const int4 eh = __ldg(tab + d.tv / 4 + d.cy + oy);
    const float l0h = __int_as_float(eh.z), l1h = __int_as_float(eh.w);
    // torch's CPU kernels: each fma rounds once; the products and the division are never contracted or reassociated
    const float w00 = __fmul_rn(l0h, l0w), w01 = __fmul_rn(l0h, l1w), w10 = __fmul_rn(l1h, l0w), w11 = __fmul_rn(l1h, l1w);
    // Direct reads: every sample of the row pair before any arithmetic, so all twelve loads are in flight at once.
    // Table reads are left to the compiler's order, which measured faster for them.
    float v[3][4], y[3];
    if constexpr (!Src::TABLE) {
#pragma unroll
      for (int c = 0; c < 3; ++c)
        v[c][0] = src(eh.x, x0, c), v[c][1] = src(eh.x, x1, c), v[c][2] = src(eh.y, x0, c), v[c][3] = src(eh.y, x1, c);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      if constexpr (Src::TABLE)
        v[c][0] = src(eh.x, x0, c), v[c][1] = src(eh.x, x1, c), v[c][2] = src(eh.y, x0, c), v[c][3] = src(eh.y, x1, c);
      const float x00 = v[c][0], x01 = v[c][1], x10 = v[c][2], x11 = v[c][3];
      if (d.form) {
        y[c] = __fmaf_rn(x11, w11, __fmaf_rn(x10, w10, __fmaf_rn(x00, w00, __fmul_rn(x01, w01))));
      } else {
        const float t0 = __fmaf_rn(x00, l0w, __fmul_rn(x01, l1w));
        const float t1 = __fmaf_rn(x10, l0w, __fmul_rn(x11, l1w));
        y[c] = __fmaf_rn(t0, l0h, __fmul_rn(t1, l1h));
      }
    }
    out(y, b, f, F, oy, ox, oh, ow);
  }
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

// The checks the clip entry points make before their launch (`who` names the entry point in the message).  A frame
// holds H W ch elements of src (src_elems counts elements); `whole`: the entry point takes no flip and no window.
static int check_clips(const char* who, const void* src, long long src_elems, int ch, bool whole,
                       const omt_clip_desc* desc, const omt_clip_desc* desc_host, const int32_t* tab,
                       const int32_t* tab_host, long long tab_len, int B, int F, int oh, int ow, const void* out) {
  OMT_REQUIRE(src && desc && desc_host && tab && tab_host && out, "%s: null pointer", who);
  OMT_REQUIRE(B >= 1 && F >= 1 && (long long)B * F <= 65535 && oh >= 1 && ow >= 1 && src_elems >= 0 && tab_len >= 0,
              "%s: B=%d, F=%d, output %dx%d, src_bytes=%lld, tab_len=%lld", who, B, F, oh, ow, src_elems, tab_len);
  for (int b = 0; b < B; ++b) {
    const omt_clip_desc& d = desc_host[b];
    OMT_REQUIRE(d.H >= 1 && d.W >= 1 && d.wh >= 1 && d.ww >= 1 && d.rh >= 1 && d.rw >= 1,
                "%s: clip %d: source %dx%d, window %dx%d, resized %dx%d", who, b, d.H, d.W, d.wh, d.ww, d.rh, d.rw);
    OMT_REQUIRE(d.src >= 0 && d.src + (long long)F * d.H * d.W * ch <= src_elems,
                "%s: clip %d: bytes [%lld, +%lld) outside the %lld source bytes", who, b, d.src,
                (long long)F * d.H * d.W * ch, src_elems);
    OMT_REQUIRE(d.y0 >= 0 && d.x0 >= 0 && (long long)d.y0 + d.wh <= d.H && (long long)d.x0 + d.ww <= d.W,
                "%s: clip %d: window %dx%d at (%d, %d) outside the %dx%d frame", who, b, d.wh, d.ww, d.y0, d.x0, d.H, d.W);
    OMT_REQUIRE(d.cy >= 0 && d.cx >= 0 && (long long)d.cy + oh <= d.rh && (long long)d.cx + ow <= d.rw,
                "%s: clip %d: crop %dx%d at (%d, %d) outside the resized %dx%d frame", who, b, oh, ow, d.cy, d.cx, d.rh,
                d.rw);
    OMT_REQUIRE((d.flip | d.form) >= 0 && (d.flip | d.form) <= 1, "%s: clip %d: flip / form must be 0 or 1", who, b);
    OMT_REQUIRE(!whole || (!d.flip && d.y0 == 0 && d.x0 == 0 && d.wh == d.H && d.ww == d.W),
                "%s: clip %d: this preprocess has no flip and no window", who, b);
    OMT_REQUIRE(clip_axis_ok(tab_host, tab_len, d.tv, d.rh, d.wh),
                "%s: clip %d: vertical table outside the table or indices outside the window", who, b);
    OMT_REQUIRE(clip_axis_ok(tab_host, tab_len, d.th, d.rw, d.ww),
                "%s: clip %d: horizontal table outside the table or indices outside the window", who, b);
  }
  return OMT_OK;
}

// The alignment checks, check_clips and the launch of one clip entry point.  `words` are its other pointers read as
// 4-byte words (fp32 sources, byte tables, sel); out is aligned to the size of what its output policy stores.
template <class Src, class Out>
static int launch_clips(const char* who, Src s, Out o, std::initializer_list<const void*> words, long long src_elems,
                        int ch, bool whole, const omt_clip_desc* desc, const omt_clip_desc* desc_host,
                        const int32_t* tab, const int32_t* tab_host, long long tab_len, int B, int F, int oh, int ow,
                        omt_stream_t stream) {
  constexpr int out_align = sizeof(*o.out);
  OMT_REQUIRE(aligned_to(8, {desc}) && aligned_to(16, {tab}) && aligned_to(out_align, {o.out}) && aligned_to(4, words),
              "%s: desc must be 8-byte, tab 16-byte, out %d-byte and tables, sel and fp32 src 4-byte aligned", who,
              out_align);
  int rc = check_clips(who, s.src, src_elems, ch, whole, desc, desc_host, tab, tab_host, tab_len, B, F, oh, ow, o.out);
  if (rc != OMT_OK) return rc;
  dim3 grid((ow + RC_TW - 1) / RC_TW, (oh + RC_TH - 1) / RC_TH, B * F);
  OMT_CUDA(launch_k(bilinear_clips_kernel<Src, Out>, grid, dim3(RC_TW), 0, (cudaStream_t)stream, s, o, desc,
                    reinterpret_cast<const int4*>(tab), F, oh, ow));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

extern "C" int omt_resample_clips(const uint8_t* src, long long src_bytes, const omt_clip_desc* desc,
                                  const omt_clip_desc* desc_host, const int32_t* tab, const int32_t* tab_host,
                                  long long tab_len, const float* norm, int B, int F, int oh, int ow, float* out,
                                  omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(norm, "omt_resample_clips: null pointer");
  return launch_clips("omt_resample_clips", ByteTable{src, norm, nullptr}, NormalizePlanes{out, norm}, {norm},
                      src_bytes, 3, false, desc, desc_host, tab, tab_host, tab_len, B, F, oh, ow, stream);
}

extern "C" int omt_fvd_preprocess(const uint8_t* src, long long src_bytes, const omt_clip_desc* desc,
                                  const omt_clip_desc* desc_host, const int32_t* tab, const int32_t* tab_host,
                                  long long tab_len, const float* lut, const int32_t* sel, int B, int F, int oh,
                                  int ow, float* out, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(lut, "omt_fvd_preprocess: null pointer");
  return launch_clips("omt_fvd_preprocess", ByteTable{src, lut, sel},
                      Float4Pixels<AFF_FVD>{reinterpret_cast<float4*>(out)}, {lut, sel}, src_bytes, 3, false, desc,
                      desc_host, tab, tab_host, tab_len, B, F, oh, ow, stream);
}

extern "C" int omt_fid_preprocess(const uint8_t* src, long long src_bytes, const omt_clip_desc* desc,
                                  const omt_clip_desc* desc_host, const int32_t* tab, const int32_t* tab_host,
                                  long long tab_len, const float* lut, const int32_t* sel, int B, int oh, int ow,
                                  float* out, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(lut, "omt_fid_preprocess: null pointer");
  return launch_clips("omt_fid_preprocess", ByteTable{src, lut, sel},
                      Float4Pixels<AFF_FID>{reinterpret_cast<float4*>(out)}, {lut, sel}, src_bytes, 3, false, desc,
                      desc_host, tab, tab_host, tab_len, B, 1, oh, ow, stream);
}

extern "C" int omt_fvd_suite_preprocess(const void* src, long long src_elems, int form, int C,
                                        const omt_clip_desc* desc, const omt_clip_desc* desc_host, const int32_t* tab,
                                        const int32_t* tab_host, long long tab_len, int B, int F, int oh, int ow,
                                        float* out, omt_stream_t stream) {
  OMT_ENTER();
  const char* who = "omt_fvd_suite_preprocess";
  OMT_REQUIRE(form == OMT_FVDS_U8 || form == OMT_FVDS_F32 || form == OMT_FVDS_F32_TRUNC, "%s: unknown input form %d",
              who, form);
  OMT_REQUIRE(form == OMT_FVDS_U8 ? C == 3 : (C == 1 || C == 3),
              "%s: C=%d (uint8 clips have 3 channels, fp32 clips 1 or 3)", who, C);
  const Float4Pixels<AFF_SUITE> o{reinterpret_cast<float4*>(out)};
  auto launch = [&](auto s) {
    return launch_clips(who, s, o, {form == OMT_FVDS_U8 ? nullptr : src}, src_elems, form == OMT_FVDS_U8 ? 3 : C,
                        true, desc, desc_host, tab, tab_host, tab_len, B, F, oh, ow, stream);
  };
  if (form == OMT_FVDS_U8) return launch(SuiteFrames<OMT_FVDS_U8>{src, C});
  if (form == OMT_FVDS_F32) return launch(SuiteFrames<OMT_FVDS_F32>{src, C});
  return launch(SuiteFrames<OMT_FVDS_F32_TRUNC>{src, C});
}

extern "C" int omt_is_preprocess(const void* src, long long src_elems, int form, const omt_clip_desc* desc,
                                 const omt_clip_desc* desc_host, const int32_t* tab, const int32_t* tab_host,
                                 long long tab_len, int B, int F, int oh, int ow, float* out, omt_stream_t stream) {
  OMT_ENTER();
  const char* who = "omt_is_preprocess";
  OMT_REQUIRE(form == OMT_FVDS_U8 || form == OMT_FVDS_F32, "%s: input form %d is neither uint8 (0) nor fp32 (1)", who,
              form);
  const Float4Pixels<AFF_NONE> o{reinterpret_cast<float4*>(out)};
  if (form == OMT_FVDS_U8)
    return launch_clips(who, SuiteFrames<OMT_FVDS_U8>{src, 3}, o, {}, src_elems, 3, true, desc, desc_host, tab,
                        tab_host, tab_len, B, F, oh, ow, stream);
  return launch_clips(who, SuiteFrames<OMT_FVDS_F32>{src, 3}, o, {src}, src_elems, 3, true, desc, desc_host, tab,
                      tab_host, tab_len, B, F, oh, ow, stream);
}

extern "C" int omt_eval_downsample(const void* src, long long src_elems, int form, const omt_clip_desc* desc,
                                   const omt_clip_desc* desc_host, const int32_t* tab, const int32_t* tab_host,
                                   long long tab_len, const float* lut, const int32_t* sel, int B, int F, int oh,
                                   int ow, uint8_t* out, omt_stream_t stream) {
  OMT_ENTER();
  const char* who = "omt_eval_downsample";
  OMT_REQUIRE(form == OMT_DS_F32 || form == OMT_DS_U8, "%s: input form %d is neither fp32 (0) nor uint8 (1)", who, form);
  OMT_REQUIRE(form == OMT_DS_F32 || lut, "%s: uint8 clips need a byte table", who);
  // a frame is H W 3 elements in both forms (3 planes of H W floats, or H W pixels of 3 bytes)
  if (form == OMT_DS_U8)
    return launch_clips(who, ByteTable{static_cast<const uint8_t*>(src), lut, sel}, BytePixels{out}, {lut, sel},
                        src_elems, 3, true, desc, desc_host, tab, tab_host, tab_len, B, F, oh, ow, stream);
  return launch_clips(who, ClampedPlanes{static_cast<const float*>(src)}, BytePixels{out}, {lut, sel, src}, src_elems,
                      3, true, desc, desc_host, tab, tab_host, tab_len, B, F, oh, ow, stream);
}
