// libjpeg-turbo's decoder arithmetic, shared by the JPEG round trip (jpeg.cu) and the JPEG decoder (jpeg_decode.cu):
// the ISLOW IDCT passes, h2v2 fancy upsampling and YCbCr -> RGB, all int32 (oracle/jpeg_oracle.py restates them).
#pragma once
#include "omt_common.cuh"

namespace omt {
namespace jpeg {

// FIX(x) = x 2^16 rounded (colour conversion), and the ISLOW DCT constants x 2^13 (CONST_BITS 13, PASS1_BITS 2)
constexpr int SCALEBITS = 16, HALF = 1 << 15;
constexpr int FIX_0_299 = 19595, FIX_0_587 = 38470, FIX_0_114 = 7471, FIX_0_16874 = 11059, FIX_0_33126 = 21709;
constexpr int FIX_0_5 = 32768, FIX_0_41869 = 27439, FIX_0_08131 = 5329;
constexpr int FIX_1_402 = 91881, FIX_0_34414 = 22554, FIX_0_71414 = 46802, FIX_1_772 = 116130;
constexpr int CONST_BITS = 13, PASS1_BITS = 2;
constexpr int F_0_298 = 2446, F_0_390 = 3196, F_0_541 = 4433, F_0_765 = 6270, F_0_899 = 7373, F_1_175 = 9633;
constexpr int F_1_501 = 12299, F_1_847 = 15137, F_1_961 = 16069, F_2_053 = 16819, F_2_562 = 20995, F_3_072 = 25172;

__device__ __forceinline__ int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }

// one pass of jpeg_idct_islow over d[0..7] in place; FIRST: the column pass on dequantised coefficients
template <bool FIRST>
__device__ __forceinline__ void idct_1d(int* d) {
  int z1 = (d[2] + d[6]) * F_0_541;
  const int tmp2e = z1 - d[6] * F_1_847, tmp3e = z1 + d[2] * F_0_765;
  const int tmp0e = (d[0] + d[4]) * (1 << CONST_BITS), tmp1e = (d[0] - d[4]) * (1 << CONST_BITS);
  const int tmp10 = tmp0e + tmp3e, tmp13 = tmp0e - tmp3e, tmp11 = tmp1e + tmp2e, tmp12 = tmp1e - tmp2e;
  int tmp0 = d[7], tmp1 = d[5], tmp2 = d[3], tmp3 = d[1];
  z1 = tmp0 + tmp3;
  int z2 = tmp1 + tmp2, z3 = tmp0 + tmp2, z4 = tmp1 + tmp3;
  const int z5 = (z3 + z4) * F_1_175;
  z1 *= -F_0_899;
  z2 *= -F_2_562;
  z3 = z3 * -F_1_961 + z5;
  z4 = z4 * -F_0_390 + z5;
  tmp0 = tmp0 * F_0_298 + z1 + z3;
  tmp1 = tmp1 * F_2_053 + z2 + z4;
  tmp2 = tmp2 * F_3_072 + z2 + z3;
  tmp3 = tmp3 * F_1_501 + z1 + z4;
  constexpr int n = FIRST ? CONST_BITS - PASS1_BITS : CONST_BITS + PASS1_BITS + 3;
  d[0] = descale(tmp10 + tmp3, n);
  d[7] = descale(tmp10 - tmp3, n);
  d[1] = descale(tmp11 + tmp2, n);
  d[6] = descale(tmp11 - tmp2, n);
  d[2] = descale(tmp12 + tmp1, n);
  d[5] = descale(tmp12 - tmp1, n);
  d[3] = descale(tmp13 + tmp0, n);
  d[4] = descale(tmp13 - tmp0, n);
}

// h2v2 fancy upsampling of chroma plane c (cs: its row stride) at output pixel (y, x); cw: the real chroma width
__device__ __forceinline__ int upsample(const uint8_t* __restrict__ c, int cs, int ch, int cw, int y, int x) {
  const int cy = y >> 1, cx = x >> 1;
  if (cw <= 2) return __ldg(c + cy * cs + cx);                 // rule (b): 2 x 2 replication
  const int ny = (y & 1) ? min(cy + 1, ch - 1) : max(cy - 1, 0);
  const uint8_t* r0 = c + cy * cs;
  const uint8_t* r1 = c + ny * cs;
  const int s = 3 * __ldg(r0 + cx) + __ldg(r1 + cx);
  if ((x & 1) == 0) {
    if (cx == 0) return (4 * s + 8) >> 4;
    return (3 * s + 3 * __ldg(r0 + cx - 1) + __ldg(r1 + cx - 1) + 8) >> 4;
  }
  if (cx == cw - 1) return (4 * s + 7) >> 4;
  return (3 * s + 3 * __ldg(r0 + cx + 1) + __ldg(r1 + cx + 1) + 7) >> 4;
}

// YCbCr -> RGB (ycc_rgb_convert's tables as arithmetic) of one pixel; cb, cr centred (minus 128)
__device__ __forceinline__ void ycc_to_rgb(int Y, int cb, int cr, uint8_t* o) {
  o[0] = (uint8_t)min(max(Y + ((FIX_1_402 * cr + HALF) >> SCALEBITS), 0), 255);
  o[1] = (uint8_t)min(max(Y + ((-FIX_0_34414 * cb - FIX_0_71414 * cr + HALF) >> SCALEBITS), 0), 255);
  o[2] = (uint8_t)min(max(Y + ((FIX_1_772 * cb + HALF) >> SCALEBITS), 0), 255);
}

}  // namespace jpeg
}  // namespace omt
