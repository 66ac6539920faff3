// The pixels of a baseline 4:2:0 JPEG save and reload, Pillow's img.save(f, "JPEG", quality=q) then
// Image.open(f).convert("RGB"), byte for byte: libjpeg-turbo's integer chain (oracle/jpeg_oracle.py restates it step by
// step).  Huffman coding is lossless, so the round trip needs no bitstream, and every step is local to a 16 x 16 MCU
// apart from the one neighbouring chroma sample the upsampling reads.
//
//   jpeg_mcu_kernel      steps 2 to 7, four horizontally adjacent MCUs per CTA: the MCU row's 16 x 64 pixels are
//                        staged in shared memory with the last row and column repeated (the padding), a thread per
//                        block row converts its 8 samples (Y, or Cb / Cr downsampled 2 x 2), runs the FDCT row pass,
//                        then the FDCT column pass, quantisation, dequantisation and the IDCT column pass on one block
//                        column, then the IDCT row pass, and writes the decoded planes to the scratch.
//   jpeg_pixel_kernel    steps 8 and 9, a thread per output pixel: h2v2 fancy upsampling of both chroma planes (plain
//                        2 x 2 replication when they are at most 2 samples wide) and YCbCr -> RGB.
//
// All arithmetic is int32; the largest intermediate of the DCTs stays below 2^28 for 8-bit samples.
#include "jpeg_common.cuh"

namespace omt {
namespace jpeg {

constexpr int MCUS = 4;                       // MCUs per CTA, side by side
constexpr int THREADS = MCUS * 6 * 8;         // a thread per block row: 4 Y blocks + Cb + Cr per MCU
constexpr int TILE_W = MCUS * 16;             // staged pixels per row
constexpr int WS = 9;                         // workspace row stride in words: conflict-free rows and columns

struct Tables {
  uint16_t q[2][64];                          // luminance, chrominance; natural order
};

// one pass of jpeg_fdct_islow over d[0..7] in place; FIRST: the row pass (outputs scaled up by 2^PASS1_BITS)
template <bool FIRST>
__device__ __forceinline__ void fdct_1d(int* d) {
  const int tmp0 = d[0] + d[7], tmp7 = d[0] - d[7], tmp1 = d[1] + d[6], tmp6 = d[1] - d[6];
  const int tmp2 = d[2] + d[5], tmp5 = d[2] - d[5], tmp3 = d[3] + d[4], tmp4 = d[3] - d[4];
  const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  constexpr int n = FIRST ? CONST_BITS - PASS1_BITS : CONST_BITS + PASS1_BITS;
  if (FIRST) {
    d[0] = (tmp10 + tmp11) * (1 << PASS1_BITS);
    d[4] = (tmp10 - tmp11) * (1 << PASS1_BITS);
  } else {
    d[0] = descale(tmp10 + tmp11, PASS1_BITS);
    d[4] = descale(tmp10 - tmp11, PASS1_BITS);
  }
  int z1 = (tmp12 + tmp13) * F_0_541;
  d[2] = descale(z1 + tmp13 * F_0_765, n);
  d[6] = descale(z1 - tmp12 * F_1_847, n);
  z1 = tmp4 + tmp7;
  int z2 = tmp5 + tmp6, z3 = tmp4 + tmp6, z4 = tmp5 + tmp7;
  const int z5 = (z3 + z4) * F_1_175;
  z1 *= -F_0_899;
  z2 *= -F_2_562;
  z3 = z3 * -F_1_961 + z5;
  z4 = z4 * -F_0_390 + z5;
  d[7] = descale(tmp4 * F_0_298 + z1 + z3, n);
  d[5] = descale(tmp5 * F_2_053 + z2 + z4, n);
  d[3] = descale(tmp6 * F_3_072 + z2 + z3, n);
  d[1] = descale(tmp7 * F_1_501 + z1 + z4, n);
}

__device__ __forceinline__ int luma(int r, int g, int b) {
  return (FIX_0_299 * r + FIX_0_587 * g + FIX_0_114 * b + HALF) >> SCALEBITS;
}
template <int COMP>   // 1: Cb, 2: Cr
__device__ __forceinline__ int chroma(int r, int g, int b) {
  if (COMP == 1) return (-FIX_0_16874 * r - FIX_0_33126 * g + FIX_0_5 * b + (128 << SCALEBITS) + HALF - 1) >> SCALEBITS;
  return (FIX_0_5 * r - FIX_0_41869 * g - FIX_0_08131 * b + (128 << SCALEBITS) + HALF - 1) >> SCALEBITS;
}
// one downsampled chroma sample from the four staged pixels at (row, col), (row, col + 1), (row + 1, ...); bias 1 or 2
template <int COMP>
__device__ __forceinline__ int chroma_2x2(const uint8_t (*px)[TILE_W * 3], int row, int col, int bias) {
  int s = bias;
#pragma unroll
  for (int dy = 0; dy < 2; ++dy)
#pragma unroll
    for (int dx = 0; dx < 2; ++dx) {
      const uint8_t* p = &px[row + dy][(col + dx) * 3];
      s += chroma<COMP>(p[0], p[1], p[2]);
    }
  return s >> 2;
}

// Scratch of one image: the Y plane (Hp x Wp), then Cb and Cr (Hp / 2 x Wp / 2), Hp and Wp the sides rounded up to 16.
__global__ void __launch_bounds__(THREADS)
jpeg_mcu_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ planes, int H, int W, int mcu_cols, int groups,
                long long items, Tables tab) {
  __shared__ uint8_t px[16][TILE_W * 3];
  __shared__ int ws[MCUS * 6][8 * WS];
  __shared__ int qt[2][64];
  const int t = threadIdx.x;
  if (t < 128) qt[t >> 6][t & 63] = tab.q[t >> 6][t & 63];
  const int Hp = ((H + 15) >> 4) << 4, Wp = ((W + 15) >> 4) << 4, ch = (H + 1) >> 1;
  const long long img_px = (long long)H * W * 3, img_planes = (long long)Hp * Wp * 3 / 2;
  // thread roles: t < 128: Y block (t >> 3) & 3 of MCU t >> 5, row t & 7; else Cb / Cr of MCU (t - 128) >> 4
  const bool is_y = t < 128;
  const int m = is_y ? t >> 5 : (t - 128) >> 4;
  const int blk = is_y ? (t >> 3) & 3 : 4 + (((t - 128) >> 3) & 1);
  const int r = t & 7;
  int* w = ws[m * 6 + blk];
  for (long long it = blockIdx.x; it < items; it += gridDim.x) {
    const int g = (int)(it % groups);
    const long long rest = it / groups;
    const int mr = (int)(rest % ((H + 15) >> 4));
    const long long b = rest / ((H + 15) >> 4);
    const uint8_t* img = src + b * img_px;
    // stage the MCU row: 16 pixel rows of 64 pixels, the last row and column repeated past the image
    __syncthreads();                       // the previous item's readers of px and ws are done
    for (int i = t; i < 16 * TILE_W * 3; i += THREADS) {
      const int row = i / (TILE_W * 3), e = i - row * (TILE_W * 3), col = e / 3;
      const int y = min(mr * 16 + row, H - 1), x = min(g * TILE_W + col, W - 1);
      px[row][e] = __ldg(img + ((long long)y * W + x) * 3 + (e - col * 3));
    }
    __syncthreads();
    // steps 2 to 4 and the FDCT row pass: this thread's 8 samples
    int d[8];
    if (is_y) {
      const int row = (blk >> 1) * 8 + r, col0 = m * 16 + (blk & 1) * 8;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const uint8_t* p = &px[row][(col0 + c) * 3];
        d[c] = luma(p[0], p[1], p[2]) - 128;
      }
    } else {
      // rule (a): rows past the image's last chroma row ceil(H / 2) - 1 repeat it
      const int row = 2 * min(r, ch - 1 - mr * 8);
#pragma unroll
      for (int c = 0; c < 8; ++c)
        d[c] = (blk == 4 ? chroma_2x2<1>(px, row, m * 16 + 2 * c, 1 + (c & 1))
                         : chroma_2x2<2>(px, row, m * 16 + 2 * c, 1 + (c & 1))) - 128;
    }
    fdct_1d<true>(d);
#pragma unroll
    for (int c = 0; c < 8; ++c) w[r * WS + c] = d[c];
    __syncthreads();
    // column r: the FDCT column pass, quantisation, dequantisation and the IDCT column pass
    const int* q = qt[blk >= 4];
#pragma unroll
    for (int k = 0; k < 8; ++k) d[k] = w[k * WS + r];
    fdct_1d<false>(d);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int qv = q[k * 8 + r], div = 8 * qv;
      const int a = (abs(d[k]) + (div >> 1)) / div;
      d[k] = (d[k] < 0 ? -a : a) * qv;
    }
    idct_1d<true>(d);
#pragma unroll
    for (int k = 0; k < 8; ++k) w[k * WS + r] = d[k];
    __syncthreads();
    // row r: the IDCT row pass, clamp(v + 128, 0, 255), one 8-byte store
#pragma unroll
    for (int c = 0; c < 8; ++c) d[c] = w[r * WS + c];
    idct_1d<false>(d);
    const int mc = g * MCUS + m;
    if (mc < mcu_cols) {
      uint32_t lo = 0, hi = 0;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        lo |= (uint32_t)min(max(d[c] + 128, 0), 255) << (8 * c);
        hi |= (uint32_t)min(max(d[c + 4] + 128, 0), 255) << (8 * c);
      }
      uint8_t* out = planes + b * img_planes;
      long long off;
      if (is_y) off = (long long)(mr * 16 + (blk >> 1) * 8 + r) * Wp + mc * 16 + (blk & 1) * 8;
      else off = (long long)Hp * Wp + (long long)(blk - 4) * (Hp / 2) * (Wp / 2) + (long long)(mr * 8 + r) * (Wp / 2) + mc * 8;
      *reinterpret_cast<uint2*>(out + off) = make_uint2(lo, hi);
    }
  }
}

__global__ void __launch_bounds__(256)
jpeg_pixel_kernel(const uint8_t* __restrict__ planes, uint8_t* __restrict__ dst, int H, int W, long long n) {
  const int Hp = ((H + 15) >> 4) << 4, Wp = ((W + 15) >> 4) << 4, ch = (H + 1) >> 1, cw = (W + 1) >> 1;
  const long long img_planes = (long long)Hp * Wp * 3 / 2;
  const long long hw = (long long)H * W;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / hw;
    const int p = (int)(i - b * hw), y = p / W, x = p - y * W;
    const uint8_t* pl = planes + b * img_planes;
    const int Y = __ldg(pl + y * Wp + x);
    const uint8_t* cbp = pl + Hp * Wp;
    const int cb = upsample(cbp, Wp / 2, ch, cw, y, x) - 128;
    const int cr = upsample(cbp + (Hp / 2) * (Wp / 2), Wp / 2, ch, cw, y, x) - 128;
    ycc_to_rgb(Y, cb, cr, dst + i * 3);
  }
}

bool overlap(const void* a, long long na, const void* b, long long nb) {
  const uintptr_t pa = reinterpret_cast<uintptr_t>(a), pb = reinterpret_cast<uintptr_t>(b);
  return pa < pb + (uintptr_t)nb && pb < pa + (uintptr_t)na;
}

}  // namespace jpeg
}  // namespace omt

using namespace omt;

extern "C" int omt_jpeg_roundtrip_u8(const uint8_t* src, uint8_t* dst, int B, int H, int W, const uint16_t* qtables,
                                     uint8_t* scratch, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(src && dst && qtables && scratch, "omt_jpeg_roundtrip_u8: null pointer");
  OMT_REQUIRE(B >= 0 && H >= 1 && W >= 1, "omt_jpeg_roundtrip_u8: B=%d images of %dx%d", B, H, W);
  jpeg::Tables tab;
  for (int i = 0; i < 128; ++i) {
    OMT_REQUIRE(qtables[i] >= 1 && qtables[i] <= 255, "omt_jpeg_roundtrip_u8: %s table entry %d is %d, outside 1..255",
                i < 64 ? "luminance" : "chrominance", i & 63, (int)qtables[i]);
    tab.q[i >> 6][i & 63] = qtables[i];
  }
  const long long Hp = ((H + 15LL) / 16) * 16, Wp = ((W + 15LL) / 16) * 16;
  OMT_REQUIRE(Hp * Wp * 3 / 2 <= 0x7fffffffLL, "omt_jpeg_roundtrip_u8: the planes of a %dx%d image overflow int32", H, W);
  OMT_REQUIRE(aligned_to(8, {scratch}), "omt_jpeg_roundtrip_u8: scratch must be 8-byte aligned");
  const long long n = (long long)B * H * W, bytes = n * 3, scratch_bytes = (long long)B * Hp * Wp * 3 / 2;
  OMT_REQUIRE(!jpeg::overlap(src, bytes, dst, bytes) && !jpeg::overlap(src, bytes, scratch, scratch_bytes) &&
              !jpeg::overlap(dst, bytes, scratch, scratch_bytes), "omt_jpeg_roundtrip_u8: src, dst and scratch overlap");
  if (B == 0) return OMT_OK;
  const cudaStream_t st = (cudaStream_t)stream;
  const int mcu_cols = (int)(Wp / 16), groups = (mcu_cols + jpeg::MCUS - 1) / jpeg::MCUS;
  const long long items = (long long)B * (Hp / 16) * groups;
  const long long cap = (long long)sm_count() * 16;
  OMT_CUDA(launch_k(jpeg::jpeg_mcu_kernel, dim3((unsigned)(items < cap ? items : cap)), dim3(jpeg::THREADS), 0, st, src,
                    scratch, H, W, mcu_cols, groups, items, tab));
  const long long blocks = (n + 255) / 256, cap2 = (long long)sm_count() * 32;
  OMT_CUDA(launch_k(jpeg::jpeg_pixel_kernel, dim3((unsigned)(blocks < cap2 ? blocks : cap2)), dim3(256), 0, st,
                    (const uint8_t*)scratch, dst, H, W, n));
  return OMT_OK;
}
