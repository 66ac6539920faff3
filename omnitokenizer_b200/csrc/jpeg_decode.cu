// Image.open(f).convert("RGB") of baseline JPEG files on the device, byte for byte as Pillow (libjpeg-turbo): the host
// parses the headers (omnitokenizer_b200/jpeg.py) and stages each file's scan and derived tables in one blob; the
// device decodes the entropy-coded data in parallel with Weissenberger & Schmidt's self-synchronising scheme (ICPP 2018)
// and runs libjpeg-turbo's integer chain (jpeg_common.cuh).  oracle/jpeg_decode_oracle.py restates every stage.
//
//   jpeg_destuff_kernel   a CTA per image: FF00 -> FF, fill bytes dropped, RSTn markers (checked in order) cut the scan
//                         into segments, the first other marker ends it (it must be EOI); each segment is cut into
//                         SUB_BITS-bit subsequences, numbered per image.
//   jpeg_sync_kernel      a CTA per GROUP subsequences, a thread per subsequence.  Each decodes its bits from an entry
//                         state (bit, block slot in the MCU, coefficient index z) to its exit state, the first symbol
//                         boundary at or past its end; inside the CTA a thread takes its predecessor's exit as its
//                         entry and decodes again until no entry changes.  Relaunches do the same across CTA
//                         boundaries until no CTA's first entry changes: each relaunch makes at least one more CTA's
//                         states right, so there are at most (CTAs per image + 1) launches, and the worst case is a
//                         serial decode of the segment, never a wrong one.  Subsequence 0 of a segment starts in the
//                         known state (its first bit, slot 0, z 0).
//   jpeg_prefix_kernel    a CTA per image: exclusive prefix sums, reset at each segment, of the per-subsequence block
//                         counts and per-component DC difference sums.
//   jpeg_coef_kernel      a thread per subsequence: decodes again from its entry, writes each block's quantised
//                         coefficients (natural order, int16, DC = prefix + differences) into serial MCU order, and
//                         checks the data: a code with no match, z > 63, a symbol past the segment's end, or more than
//                         7 bits left after the segment's last block set the image's status word.
//   jpeg_idct_kernel      8 threads per block: dequantise, ISLOW IDCT into padded component planes.
//   jpeg_rgb_kernel       a thread per pixel: fancy upsampling (h2v1, h2v2) and YCbCr -> RGB, or grey replicated, into
//                         the packed (H, W, 3) output; one thread per image also checks every segment was completed.
#include <algorithm>

#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include "jpeg_common.cuh"

namespace omt {
namespace jdec {

using namespace omt::jpeg;

constexpr int GROUP = 128;              // subsequences per sync / coefficient CTA
constexpr int SUB_BITS = 1024;          // bits per subsequence
constexpr int THREADS = 256;            // destuff, prefix, IDCT and pixel CTAs
constexpr int BYTES_PER_THREAD = 16;    // destuff: bytes each thread classifies per tile
constexpr int TILE = THREADS * BYTES_PER_THREAD;

enum Status { OK = 0, NO_END = 1, RST_ORDER = 2, RST_COUNT = 3, BAD_CODE = 4, BAD_Z = 5, SHORT = 6, NOT_EOI = 7, EXTRA = 8 };

__constant__ uint8_t kNatural[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                     41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                     30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// ------------------------------------------------------------------------------------------------ geometry and layout
struct Geo {
  int hmax, vmax, mx, my, bpm, nseg, mcus;
  int pw[3], ph[3];     // component plane sizes: the whole MCU grid
};

__host__ __device__ inline Geo geo_of(const omt_jpeg_desc& d) {
  Geo g;
  g.hmax = g.vmax = 1;
  for (int c = 0; c < d.ncomp; ++c) {
    g.hmax = max(g.hmax, d.h[c]);
    g.vmax = max(g.vmax, d.v[c]);
  }
  g.mx = (d.W + 8 * g.hmax - 1) / (8 * g.hmax);
  g.my = (d.H + 8 * g.vmax - 1) / (8 * g.vmax);
  g.mcus = g.mx * g.my;
  g.bpm = 0;
  for (int c = 0; c < 3; ++c) {
    const bool on = c < d.ncomp;
    g.pw[c] = on ? g.mx * d.h[c] * 8 : 0;
    g.ph[c] = on ? g.my * d.v[c] * 8 : 0;
    g.bpm += on ? d.h[c] * d.v[c] : 0;
  }
  g.nseg = d.restart > 0 ? (g.mcus + d.restart - 1) / d.restart : 1;
  return g;
}

// Byte offsets inside an image's work area (omnitokenizer_b200/jpeg.py work_bytes restates them).
struct Work {
  long long segs, sbase, data, entry, exitp, cnt, pre, coef, plane[3], bytes;
};

__host__ __device__ inline long long up256(long long x) { return (x + 255) & ~255LL; }

__host__ __device__ inline Work work_of(const omt_jpeg_desc& d, const Geo& g) {
  Work w;
  long long o = 256;                                   // int32 counters: segments found, subsequences, segments done
  w.segs = o;  o = up256(o + 4LL * (g.nseg + 1));      // destuffed byte offset of each segment, then the end
  w.sbase = o; o = up256(o + 4LL * (g.nseg + 1));      // first subsequence of each segment, then the count
  w.data = o;  o = up256(o + d.scan_bytes + 16);       // destuffed bytes, zero padded for the bit reader
  w.entry = o; o += 8LL * d.nsub;                      // packed states
  w.exitp = o; o += 8LL * d.nsub;
  w.cnt = o;   o += 16LL * d.nsub;                     // blocks started, DC difference sums per component
  w.pre = o;   o += 16LL * d.nsub;                     // their exclusive prefix within the segment
  w.coef = o;  o = up256(o + 128LL * g.mcus * g.bpm);  // int16 [blocks][64]
  for (int c = 0; c < 3; ++c) {
    w.plane[c] = o;
    o = up256(o + (long long)g.pw[c] * g.ph[c]);
  }
  w.bytes = o;
  return w;
}

enum Hdr { H_FOUND = 0, H_NSUB = 1, H_DONE = 2 };

__device__ __forceinline__ void set_status(int32_t* status, int code) { atomicCAS(status, 0, code); }

// ------------------------------------------------------------------------------------------------ tables in shared memory
struct SmemTables {
  uint16_t lut[6][256];
  int maxcode[6][18];
  int valoff[6][18];
  uint8_t val[6][256];
  int8_t slot_comp[8];
};

__device__ void load_tables(SmemTables& s, const omt_jpeg_tables* t, const omt_jpeg_desc& d) {
  const int n = 2 * d.ncomp;
  for (int i = threadIdx.x; i < n * 256; i += blockDim.x) {
    s.lut[i >> 8][i & 255] = t->lookup[i >> 8][i & 255];
    s.val[i >> 8][i & 255] = t->values[i >> 8][i & 255];
  }
  for (int i = threadIdx.x; i < n * 18; i += blockDim.x) {
    s.maxcode[i / 18][i % 18] = t->maxcode[i / 18][i % 18];
    s.valoff[i / 18][i % 18] = t->valoffset[i / 18][i % 18];
  }
  if (threadIdx.x == 0) {
    int k = 0;
    for (int c = 0; c < d.ncomp; ++c)
      for (int i = 0; i < d.h[c] * d.v[c]; ++i) s.slot_comp[k++] = (int8_t)c;
  }
}

// ------------------------------------------------------------------------------------------------ the symbol decoder
struct St {
  unsigned pos;
  int slot, z;     // z = 0: the next symbol is a block's DC one
};
__device__ __forceinline__ unsigned long long pack(const St& s) {
  return (unsigned long long)s.pos << 16 | (unsigned)(s.slot << 8) | (unsigned)s.z;
}
__device__ __forceinline__ St unpack(unsigned long long v) {
  return St{(unsigned)(v >> 16), (int)(v >> 8) & 255, (int)v & 255};
}

// 32 bits of the big-endian stream from bit pos
__device__ __forceinline__ uint32_t peek32(const uint32_t* __restrict__ w, unsigned pos) {
  const unsigned i = pos >> 5;
  const uint32_t hi = __byte_perm(__ldg(w + i), 0, 0x0123), lo = __byte_perm(__ldg(w + i + 1), 0, 0x0123);
  return __funnelshift_l(lo, hi, pos & 31);
}

__device__ __forceinline__ void end_block(St& s, int bpm) {
  s.z = 0;
  s.slot = s.slot + 1 == bpm ? 0 : s.slot + 1;
}

// One symbol from state s.  Returns 1 for a DC symbol (val: the difference), 2 for a coefficient (k: its zigzag index,
// val), 0 for a run of zeros or EOB, -status for an error, which ends the block so that speculative decoding stays
// deterministic (oracle/jpeg_decode_oracle.py step).
__device__ __forceinline__ int step(const SmemTables& T, int bpm, const uint32_t* __restrict__ data, St& s, int& k,
                                    int& val) {
  const int t = 2 * T.slot_comp[s.slot] + (s.z != 0);
  const uint32_t w = peek32(data, s.pos);
  int len = 0, sym = 0;
  const int e = T.lut[t][w >> 24];
  if ((e >> 8) <= 8) {
    len = e >> 8;
    sym = e & 255;
  } else {
#pragma unroll 1
    for (int l = 9; l <= 16; ++l) {
      const int code = (int)(w >> (32 - l));
      if (code <= T.maxcode[t][l]) {
        len = l;
        sym = T.val[t][(code + T.valoff[t][l]) & 255];
        break;
      }
    }
  }
  if (len == 0 || (s.z == 0 && sym > 15)) {
    s.pos += 16;
    end_block(s, bpm);
    return -BAD_CODE;
  }
  const int sz = sym & 15, r = s.z == 0 ? 0 : sym >> 4;
  val = 0;
  if (sz) {
    const uint32_t bits = (w << len) >> (32 - sz);
    val = bits < (1u << (sz - 1)) ? (int)bits - (1 << sz) + 1 : (int)bits;
  }
  s.pos += len + sz;
  if (s.z == 0) {
    s.z = 1;
    return 1;
  }
  if (sz) {
    k = s.z + r;
    if (k > 63) {
      end_block(s, bpm);
      return -BAD_Z;
    }
    s.z = k + 1;
    if (s.z == 64) end_block(s, bpm);
    return 2;
  }
  if (r == 15) {
    if (s.z + 16 > 64) {
      end_block(s, bpm);
      return -BAD_Z;
    }
    s.z += 16;
    if (s.z == 64) end_block(s, bpm);
    return 0;
  }
  end_block(s, bpm);
  return 0;
}

// the segment holding subsequence s: the last k with sbase[k] <= s
__device__ __forceinline__ int segment_of(const int* sbase, int nseg, int s) {
  int lo = 0, hi = nseg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (sbase[mid] <= s) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// ------------------------------------------------------------------------------------------------ destuff
__global__ void __launch_bounds__(THREADS)
jpeg_destuff_kernel(const uint8_t* __restrict__ blob, const omt_jpeg_desc* __restrict__ desc, uint8_t* __restrict__ scratch,
                    int32_t* __restrict__ status) {
  using Scan = cub::BlockScan<int2, THREADS>;
  using Reduce = cub::BlockReduce<long long, THREADS>;
  __shared__ union {
    typename Scan::TempStorage scan;
    typename Reduce::TempStorage reduce;
  } tmp;
  __shared__ long long s_end;
  __shared__ int2 s_tot;
  const int b = blockIdx.x, t = threadIdx.x;
  const omt_jpeg_desc d = desc[b];
  const Geo g = geo_of(d);
  const Work wk = work_of(d, g);
  uint8_t* work = scratch + d.work;
  int* hdr = reinterpret_cast<int*>(work);
  int* segs = reinterpret_cast<int*>(work + wk.segs);
  int* sbase = reinterpret_cast<int*>(work + wk.sbase);
  uint8_t* out = work + wk.data;
  const uint8_t* src = blob + d.scan;
  const long long n = d.scan_bytes;
  const long long NONE = 0x7fffffffffffffffLL;
  int out_pos = 0, rst = 0;                 // carried across tiles (uniform)
  long long end = NONE;
  bool bad_order = false, too_many = false;
  for (long long base = 0; base < n && end == NONE; base += TILE) {
    const long long j0 = base + (long long)t * BYTES_PER_THREAD;
    // the first byte of a marker other than RSTn, or of an FF at the very end
    long long e = NONE;
    for (int i = 0; i < BYTES_PER_THREAD; ++i) {
      const long long j = j0 + i;
      if (j >= n) break;
      if (src[j] == 0xFF) {
        const int nx = j + 1 < n ? src[j + 1] : -1;
        if (nx != 0x00 && nx != 0xFF && !(nx >= 0xD0 && nx <= 0xD7)) {
          e = j;
          break;
        }
      }
    }
    const long long te = Reduce(tmp.reduce).Reduce(e, cub::Min());
    if (t == 0) s_end = te;
    __syncthreads();
    const long long lim = s_end < n ? s_end : n;
    // count the kept bytes and RST markers below lim, then write them
    int2 c = make_int2(0, 0);
    for (int i = 0; i < BYTES_PER_THREAD; ++i) {
      const long long j = j0 + i;
      if (j >= lim) break;
      const int v = src[j];
      if (v == 0xFF) {
        const int nx = src[j + 1];
        c.x += nx == 0x00;
        c.y += nx >= 0xD0 && nx <= 0xD7;
      } else if (j == 0 || src[j - 1] != 0xFF) {
        c.x += 1;
      }
    }
    int2 pre, tot;
    Scan(tmp.scan).ExclusiveScan(c, pre, make_int2(0, 0),
                                 [](int2 a, int2 b2) { return make_int2(a.x + b2.x, a.y + b2.y); }, tot);
    int o = out_pos + pre.x, r = rst + pre.y;
    for (int i = 0; i < BYTES_PER_THREAD; ++i) {
      const long long j = j0 + i;
      if (j >= lim) break;
      const int v = src[j];
      if (v == 0xFF) {
        const int nx = src[j + 1];
        if (nx == 0x00) {
          out[o++] = 0xFF;
        } else if (nx >= 0xD0 && nx <= 0xD7) {
          if (nx != 0xD0 + (r & 7)) bad_order = true;
          if (r + 1 < g.nseg) segs[r + 1] = o;
          else too_many = true;
          ++r;
        }
      } else if (j == 0 || src[j - 1] != 0xFF) {
        out[o++] = (uint8_t)v;
      }
    }
    if (t == 0) s_tot = tot;
    __syncthreads();
    out_pos += s_tot.x;
    rst += s_tot.y;
    end = s_end;
    __syncthreads();                        // s_end, s_tot and tmp are reused by the next tile
  }
  const bool any_bad_order = __syncthreads_or(bad_order);
  if (t != 0) return;
  int code = OK;
  if (any_bad_order) code = RST_ORDER;
  else if (end == NONE || end + 1 >= n) code = NO_END;
  else if (src[end + 1] != 0xD9) code = NOT_EOI;
  else if (too_many || rst + 1 != g.nseg) code = RST_COUNT;
  if (code != OK) {
    set_status(status + b, code);
    hdr[H_FOUND] = 0;
    hdr[H_NSUB] = 0;                        // nothing of this image is decoded
    return;
  }
  segs[0] = 0;
  segs[g.nseg] = out_pos;
  int s = 0;
  for (int k = 0; k < g.nseg; ++k) {      // one thread: the segment count is at most the MCU count
    sbase[k] = s;
    s += (8 * (segs[k + 1] - segs[k]) + SUB_BITS - 1) / SUB_BITS;
  }
  sbase[g.nseg] = s;
  hdr[H_FOUND] = g.nseg;
  hdr[H_NSUB] = s;
}

// ------------------------------------------------------------------------------------------------ synchronisation
struct Sub {
  int k, i;                 // segment, index in it
  unsigned start, end, seg_end;
};

__device__ __forceinline__ Sub sub_of(const uint8_t* work, const Work& wk, int nseg, int s) {
  const int* segs = reinterpret_cast<const int*>(work + wk.segs);
  const int* sbase = reinterpret_cast<const int*>(work + wk.sbase);
  Sub u;
  u.k = segment_of(sbase, nseg, s);
  u.i = s - sbase[u.k];
  u.seg_end = 8u * (unsigned)segs[u.k + 1];
  u.start = 8u * (unsigned)segs[u.k] + (unsigned)u.i * SUB_BITS;
  u.end = min(u.start + SUB_BITS, u.seg_end);
  return u;
}

// decode [entry, end): the exit state, blocks started and DC difference sums per component
__device__ __forceinline__ void run_sub(const SmemTables& T, int bpm, const uint32_t* data, unsigned long long entry,
                                        unsigned end, unsigned long long& exit_state, int4& cnt) {
  St s = unpack(entry);
  int4 c = make_int4(0, 0, 0, 0);
  while (s.pos < end) {
    const int comp = T.slot_comp[s.slot];
    int k, v;
    if (step(T, bpm, data, s, k, v) == 1) {
      c.x += 1;
      c.y += comp == 0 ? v : 0;
      c.z += comp == 1 ? v : 0;
      c.w += comp == 2 ? v : 0;
    }
  }
  exit_state = pack(s);
  cnt = c;
}

__global__ void __launch_bounds__(GROUP)
jpeg_sync_kernel(const uint8_t* __restrict__ blob, const omt_jpeg_desc* __restrict__ desc, uint8_t* __restrict__ scratch,
                 int first) {
  __shared__ SmemTables T;
  __shared__ unsigned long long ex[GROUP];
  __shared__ int go;
  const int b = blockIdx.y, t = threadIdx.x;
  const omt_jpeg_desc d = desc[b];
  const Geo g = geo_of(d);
  const Work wk = work_of(d, g);
  uint8_t* work = scratch + d.work;
  const int* hdr = reinterpret_cast<const int*>(work);
  const int nsub = hdr[H_NSUB], s0 = blockIdx.x * GROUP, s = s0 + t;
  if (s0 >= nsub) return;
  const bool active = s < nsub;
  unsigned long long* entry = reinterpret_cast<unsigned long long*>(work + wk.entry);
  unsigned long long* exitp = reinterpret_cast<unsigned long long*>(work + wk.exitp);
  int4* cnt = reinterpret_cast<int4*>(work + wk.cnt);
  int* changed = reinterpret_cast<int*>(scratch);
  const Sub u = sub_of(work, wk, hdr[H_FOUND], active ? s : s0);
  unsigned long long my_entry = 0, my_exit = 0;
  int4 my_cnt = make_int4(0, 0, 0, 0);
  bool redo;
  if (first) {
    my_entry = pack(St{u.start, 0, 0});
    redo = active;
  } else {
    // relaunch: only a CTA whose first entry differs from its predecessor's exit decodes again
    if (t == 0) {
      go = 0;
      if (u.i != 0) {
        const unsigned long long e = __ldcg(exitp + s0 - 1);
        if (e != entry[s0]) {
          go = 1;
          atomicExch(changed, 1);
        }
      }
    }
    __syncthreads();
    if (!go) return;
    if (active) {
      my_entry = entry[s];
      my_exit = exitp[s];
      my_cnt = cnt[s];
    }
    redo = t == 0;
    if (redo) my_entry = __ldcg(exitp + s0 - 1);
  }
  load_tables(T, reinterpret_cast<const omt_jpeg_tables*>(blob + d.tables), d);
  __syncthreads();
  const uint32_t* data = reinterpret_cast<const uint32_t*>(work + wk.data);
  for (;;) {
    if (redo) run_sub(T, g.bpm, data, my_entry, u.end, my_exit, my_cnt);
    ex[t] = my_exit;
    __syncthreads();
    redo = false;
    if (active && t > 0 && u.i != 0 && ex[t - 1] != my_entry) {
      my_entry = ex[t - 1];
      redo = true;
    }
    if (!__syncthreads_or(redo)) break;
  }
  if (active) {
    entry[s] = my_entry;
    __stcg(exitp + s, my_exit);
    cnt[s] = my_cnt;
  }
}

// ------------------------------------------------------------------------------------------------ prefix sums
struct SegSum {
  int head;
  int4 v;
};

__global__ void __launch_bounds__(THREADS)
jpeg_prefix_kernel(const omt_jpeg_desc* __restrict__ desc, uint8_t* __restrict__ scratch) {
  using Scan = cub::BlockScan<SegSum, THREADS>;
  __shared__ typename Scan::TempStorage tmp;
  const int b = blockIdx.x, t = threadIdx.x;
  const omt_jpeg_desc d = desc[b];
  const Geo g = geo_of(d);
  const Work wk = work_of(d, g);
  uint8_t* work = scratch + d.work;
  const int* hdr = reinterpret_cast<const int*>(work);
  const int nsub = hdr[H_NSUB], nseg = hdr[H_FOUND];
  const int* sbase = reinterpret_cast<const int*>(work + wk.sbase);
  const int4* cnt = reinterpret_cast<const int4*>(work + wk.cnt);
  int4* pre = reinterpret_cast<int4*>(work + wk.pre);
  auto op = [](const SegSum& a, const SegSum& c) {
    return c.head ? c : SegSum{a.head, make_int4(a.v.x + c.v.x, a.v.y + c.v.y, a.v.z + c.v.z, a.v.w + c.v.w)};
  };
  SegSum carry{0, make_int4(0, 0, 0, 0)};
  for (int base = 0; base < nsub; base += THREADS) {
    const int s = base + t;
    SegSum x{1, make_int4(0, 0, 0, 0)};
    if (s < nsub) {
      x.v = cnt[s];
      x.head = sbase[segment_of(sbase, nseg, s)] == s;
    }
    SegSum incl, agg;
    Scan(tmp).InclusiveScan(x, incl, op, agg);
    const SegSum tot = op(carry, incl);
    if (s < nsub) {
      const int4 v = x.v, a = tot.v;
      pre[s] = make_int4(a.x - v.x, a.y - v.y, a.z - v.z, a.w - v.w);
    }
    carry = op(carry, agg);
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------ coefficients
__global__ void __launch_bounds__(GROUP)
jpeg_coef_kernel(const uint8_t* __restrict__ blob, const omt_jpeg_desc* __restrict__ desc, uint8_t* __restrict__ scratch,
                 int32_t* __restrict__ status) {
  __shared__ SmemTables T;
  const int b = blockIdx.y, t = threadIdx.x;
  const omt_jpeg_desc d = desc[b];
  const Geo g = geo_of(d);
  const Work wk = work_of(d, g);
  uint8_t* work = scratch + d.work;
  int* hdr = reinterpret_cast<int*>(work);
  const int nsub = hdr[H_NSUB], s = blockIdx.x * GROUP + t;
  if (blockIdx.x * GROUP >= nsub) return;
  load_tables(T, reinterpret_cast<const omt_jpeg_tables*>(blob + d.tables), d);
  __syncthreads();
  if (s >= nsub) return;
  const Sub u = sub_of(work, wk, hdr[H_FOUND], s);
  const int4 p = reinterpret_cast<const int4*>(work + wk.pre)[s];
  const int per = d.restart > 0 ? d.restart : g.mcus;
  const int seg_blocks = min(per, g.mcus - u.k * per) * g.bpm;
  St st = unpack(reinterpret_cast<const unsigned long long*>(work + wk.entry)[s]);
  int started = p.x;
  if (started > seg_blocks || (started == seg_blocks && st.z == 0)) return;     // past the segment's last block
  int16_t* coef = reinterpret_cast<int16_t*>(work + wk.coef);
  const uint32_t* data = reinterpret_cast<const uint32_t*>(work + wk.data);
  long long block = (long long)u.k * per * g.bpm + started - 1;                 // the block in progress
  int dc0 = p.y, dc1 = p.z, dc2 = p.w;
  while (st.pos < u.end) {
    const int comp = T.slot_comp[st.slot];
    int k, v;
    const int ev = step(T, g.bpm, data, st, k, v);
    if (st.pos > u.seg_end) {
      set_status(status + b, SHORT);
      return;
    }
    if (ev < 0) {
      set_status(status + b, -ev);
      return;
    }
    if (ev == 1) {
      ++block;
      ++started;
      const int dc = comp == 0 ? (dc0 += v) : comp == 1 ? (dc1 += v) : (dc2 += v);
      coef[block * 64] = (int16_t)dc;
    } else if (ev == 2) {
      coef[block * 64 + kNatural[k]] = (int16_t)v;
    }
    if (st.z == 0 && started == seg_blocks) {
      if (u.seg_end - st.pos >= 8) set_status(status + b, EXTRA);
      else atomicAdd(hdr + H_DONE, 1);
      return;
    }
  }
}

// ------------------------------------------------------------------------------------------------ IDCT
constexpr int IDCT_BLOCKS = THREADS / 8;
constexpr int WS = 9;

__global__ void __launch_bounds__(THREADS)
jpeg_idct_kernel(const uint8_t* __restrict__ blob, const omt_jpeg_desc* __restrict__ desc, uint8_t* __restrict__ scratch) {
  __shared__ int q[3][64];
  __shared__ int ws[IDCT_BLOCKS][8 * WS];
  const int b = blockIdx.y, t = threadIdx.x;
  const omt_jpeg_desc d = desc[b];
  const Geo g = geo_of(d);
  const Work wk = work_of(d, g);
  const uint8_t* work = scratch + d.work;
  const omt_jpeg_tables* tab = reinterpret_cast<const omt_jpeg_tables*>(blob + d.tables);
  for (int i = t; i < d.ncomp * 64; i += THREADS) q[i >> 6][i & 63] = tab->q[i >> 6][i & 63];
  const int16_t* coef = reinterpret_cast<const int16_t*>(work + wk.coef);
  const int nblocks = g.mcus * g.bpm, lb = t >> 3, r = t & 7;
  int* w = ws[lb];
  for (int base = blockIdx.x * IDCT_BLOCKS; base < nblocks; base += gridDim.x * IDCT_BLOCKS) {
    __syncthreads();                     // q is loaded; the previous round's rows are read
    const int j = base + lb;
    const bool valid = j < nblocks;
    const int mcu = valid ? j / g.bpm : 0, slot = j - mcu * g.bpm;
    int c = 0, first = 0;
    while (c + 1 < d.ncomp && slot >= first + d.h[c] * d.v[c]) first += d.h[c] * d.v[c], ++c;
    int dv[8];
    if (valid) {
      const int16_t* blk = coef + (long long)j * 64;
#pragma unroll
      for (int k = 0; k < 8; ++k) dv[k] = (int)blk[k * 8 + r] * q[c][k * 8 + r];
      idct_1d<true>(dv);
#pragma unroll
      for (int k = 0; k < 8; ++k) w[k * WS + r] = dv[k];
    }
    __syncthreads();
    if (valid) {
#pragma unroll
      for (int k = 0; k < 8; ++k) dv[k] = w[r * WS + k];
      idct_1d<false>(dv);
      uint32_t lo = 0, hi = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        lo |= (uint32_t)min(max(dv[k] + 128, 0), 255) << (8 * k);
        hi |= (uint32_t)min(max(dv[k + 4] + 128, 0), 255) << (8 * k);
      }
      const int in = slot - first, by = in / d.h[c], bx = in - by * d.h[c];
      const int my = mcu / g.mx, mx = mcu - my * g.mx;
      const long long row = (long long)(my * d.v[c] + by) * 8 + r, col = (long long)(mx * d.h[c] + bx) * 8;
      *reinterpret_cast<uint2*>(scratch + d.work + wk.plane[c] + row * g.pw[c] + col) = make_uint2(lo, hi);
    }
  }
}

// ------------------------------------------------------------------------------------------------ pixels
// h2v1 fancy upsampling of row c at output column x; cw: the real chroma width
__device__ __forceinline__ int upsample_h2v1(const uint8_t* __restrict__ c, int cw, int x) {
  const int cx = x >> 1;
  const int v = __ldg(c + cx);
  if (cw <= 2) return v;
  if ((x & 1) == 0) return cx == 0 ? v : (3 * v + __ldg(c + cx - 1) + 1) >> 2;
  return cx == cw - 1 ? v : (3 * v + __ldg(c + cx + 1) + 2) >> 2;
}

__global__ void __launch_bounds__(THREADS)
jpeg_rgb_kernel(const omt_jpeg_desc* __restrict__ desc, const uint8_t* __restrict__ scratch, uint8_t* __restrict__ out,
                int32_t* __restrict__ status) {
  const int b = blockIdx.y;
  const omt_jpeg_desc d = desc[b];
  const Geo g = geo_of(d);
  const Work wk = work_of(d, g);
  const uint8_t* work = scratch + d.work;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const int* hdr = reinterpret_cast<const int*>(work);
    if (hdr[H_FOUND] != g.nseg || hdr[H_DONE] != g.nseg) set_status(status + b, SHORT);
  }
  const uint8_t* py = work + wk.plane[0];
  const uint8_t* pcb = work + wk.plane[1];
  const uint8_t* pcr = work + wk.plane[2];
  const int W = d.W, cw = (W * d.h[1] + g.hmax - 1) / g.hmax, ch = (d.H * d.v[1] + g.vmax - 1) / g.vmax;
  const long long n = (long long)d.H * W;
  uint8_t* o = out + d.out;
  for (long long i = blockIdx.x * (long long)THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * THREADS) {
    const int y = (int)(i / W), x = (int)(i - (long long)y * W);
    const int Y = __ldg(py + (long long)y * g.pw[0] + x);
    if (d.ncomp == 1) {
      o[i * 3] = o[i * 3 + 1] = o[i * 3 + 2] = (uint8_t)Y;
      continue;
    }
    int cb, cr;
    if (g.hmax == 1) {
      cb = __ldg(pcb + (long long)y * g.pw[1] + x);
      cr = __ldg(pcr + (long long)y * g.pw[2] + x);
    } else if (g.vmax == 1) {
      cb = upsample_h2v1(pcb + (long long)y * g.pw[1], cw, x);
      cr = upsample_h2v1(pcr + (long long)y * g.pw[2], cw, x);
    } else {
      cb = upsample(pcb, g.pw[1], ch, cw, y, x);
      cr = upsample(pcr, g.pw[2], ch, cw, y, x);
    }
    ycc_to_rgb(Y, cb - 128, cr - 128, o + i * 3);
  }
}

bool overlap(const void* a, long long na, const void* b, long long nb) {
  const uintptr_t pa = reinterpret_cast<uintptr_t>(a), pb = reinterpret_cast<uintptr_t>(b);
  return na > 0 && nb > 0 && pa < pb + (uintptr_t)nb && pb < pa + (uintptr_t)na;
}

int decode(const uint8_t* blob, long long blob_bytes, const omt_jpeg_desc* desc, const omt_jpeg_desc* desc_host, int B,
           uint8_t* scratch, long long scratch_bytes, uint8_t* out, long long out_bytes, int32_t* status,
           float* stage_ms, int* sync_launches, omt_stream_t stream) {
  const char* who = "omt_jpeg_decode_u8";
  OMT_REQUIRE(B >= 0 && B <= 65535, "%s: B=%d images unsupported (0..65535)", who, B);
  if (B == 0) return OMT_OK;
  OMT_REQUIRE(blob && desc && desc_host && scratch && out && status, "%s: null pointer", who);
  OMT_REQUIRE(aligned_to(16, {blob}) && aligned_to(256, {scratch}), "%s: blob must be 16-byte and scratch 256-byte aligned",
              who);
  OMT_REQUIRE(!overlap(blob, blob_bytes, scratch, scratch_bytes) && !overlap(blob, blob_bytes, out, out_bytes) &&
                  !overlap(scratch, scratch_bytes, out, out_bytes) && !overlap(status, 4LL * B, out, out_bytes) &&
                  !overlap(status, 4LL * B, scratch, scratch_bytes),
              "%s: blob, scratch, out and status overlap", who);
  long long next = 256;       // the first 256 scratch bytes hold the synchronisation flag
  int groups = 0;
  for (int b = 0; b < B; ++b) {
    const omt_jpeg_desc& d = desc_host[b];
    OMT_REQUIRE(d.H >= 1 && d.H <= 65535 && d.W >= 1 && d.W <= 65535, "%s: image %d is %dx%d", who, b, d.H, d.W);
    OMT_REQUIRE(d.ncomp == 1 || d.ncomp == 3, "%s: image %d has %d components (1 or 3)", who, b, d.ncomp);
    const bool gray = d.ncomp == 1 && d.h[0] == 1 && d.v[0] == 1;
    const bool ycc = d.ncomp == 3 && ((d.h[0] == 1 && d.v[0] == 1) || (d.h[0] == 2 && d.v[0] == 1) ||
                                      (d.h[0] == 2 && d.v[0] == 2)) &&
                     d.h[1] == 1 && d.v[1] == 1 && d.h[2] == 1 && d.v[2] == 1;
    OMT_REQUIRE(gray || ycc, "%s: image %d: sampling factors not 1x1 (grey) or 1x1 / 2x1 / 2x2 with 1x1 chroma", who, b);
    OMT_REQUIRE(d.restart >= 0 && d.restart <= 65535, "%s: image %d: restart interval %d", who, b, d.restart);
    OMT_REQUIRE(d.scan >= 0 && d.scan_bytes >= 1 && d.scan_bytes <= (1LL << 27) && d.scan + d.scan_bytes <= blob_bytes,
                "%s: image %d: scan [%lld, +%lld) is not inside the %lld-byte blob (at most 2^27 bytes)", who, b, d.scan,
                d.scan_bytes, blob_bytes);
    OMT_REQUIRE(d.tables >= 0 && d.tables % 16 == 0 && d.tables + (long long)sizeof(omt_jpeg_tables) <= blob_bytes,
                "%s: image %d: tables at %lld are not a 16-byte aligned omt_jpeg_tables inside the blob", who, b,
                d.tables);
    const long long px = 3LL * d.H * d.W;
    OMT_REQUIRE(d.out >= 0 && d.out + px <= out_bytes, "%s: image %d: output [%lld, +%lld) is not inside the %lld-byte out",
                who, b, d.out, px, out_bytes);
    const Geo g = geo_of(d);
    const long long need = (8 * d.scan_bytes + SUB_BITS - 1) / SUB_BITS + g.nseg;
    OMT_REQUIRE(d.nsub % GROUP == 0 && d.nsub >= need && d.nsub <= need + GROUP,
                "%s: image %d: %d subsequence slots, expected %lld rounded up to a multiple of %d", who, b, d.nsub, need,
                GROUP);
    const Work wk = work_of(d, g);
    OMT_REQUIRE(d.work % 256 == 0 && d.work >= next && d.work + wk.bytes <= scratch_bytes,
                "%s: image %d: work area [%lld, +%lld) is not 256-byte aligned, after the previous one and inside the "
                "%lld-byte scratch", who, b, d.work, wk.bytes, scratch_bytes);
    next = d.work + wk.bytes;
    groups = max(groups, d.nsub / GROUP);
  }
  const cudaStream_t st = (cudaStream_t)stream;
  struct Events {             // destroyed on every return, early ones included
    cudaEvent_t e[6];
    int n = 0;
    ~Events() {
      for (int i = 0; i < n; ++i) cudaEventDestroy(e[i]);
    }
  } ev;
  if (stage_ms)
    for (; ev.n < 6; ++ev.n) OMT_CUDA(cudaEventCreate(&ev.e[ev.n]));
  auto mark = [&](int i) { return stage_ms ? cudaEventRecord(ev.e[i], st) : cudaSuccess; };
  OMT_CUDA(mark(0));
  OMT_CUDA(cudaMemsetAsync(scratch, 0, next, st));
  OMT_CUDA(cudaMemsetAsync(status, 0, 4LL * B, st));
  OMT_CUDA(launch_k(jpeg_destuff_kernel, dim3(B), dim3(THREADS), 0, st, blob, desc, scratch, status));
  OMT_CUDA(mark(1));
  const dim3 grid_sub(groups, B);
  OMT_CUDA(launch_k(jpeg_sync_kernel, grid_sub, dim3(GROUP), 0, st, blob, desc, scratch, 1));
  int launches = 1;
  for (;;) {
    int changed = 0;
    OMT_CUDA(cudaMemsetAsync(scratch, 0, 4, st));
    OMT_CUDA(launch_k(jpeg_sync_kernel, grid_sub, dim3(GROUP), 0, st, blob, desc, scratch, 0));
    ++launches;
    OMT_CUDA(cudaMemcpyAsync(&changed, scratch, 4, cudaMemcpyDeviceToHost, st));
    OMT_CUDA(cudaStreamSynchronize(st));
    if (!changed) break;
    OMT_REQUIRE(launches <= groups + 2, "%s: the synchronisation did not settle in %d launches", who, launches);
  }
  OMT_CUDA(mark(2));
  OMT_CUDA(launch_k(jpeg_prefix_kernel, dim3(B), dim3(THREADS), 0, st, desc, scratch));
  OMT_CUDA(launch_k(jpeg_coef_kernel, grid_sub, dim3(GROUP), 0, st, blob, desc, scratch, status));
  OMT_CUDA(mark(3));
  long long max_blocks = 0, max_px = 0;
  for (int b = 0; b < B; ++b) {
    const Geo g = geo_of(desc_host[b]);
    max_blocks = std::max(max_blocks, (long long)g.mcus * g.bpm);
    max_px = std::max(max_px, (long long)desc_host[b].H * desc_host[b].W);
  }
  const long long cap = (long long)sm_count() * 8;
  const long long gi = (max_blocks + IDCT_BLOCKS - 1) / IDCT_BLOCKS, gp = (max_px + THREADS - 1) / THREADS;
  OMT_CUDA(launch_k(jpeg_idct_kernel, dim3((unsigned)std::min(gi, cap), B), dim3(THREADS), 0, st, blob, desc, scratch));
  OMT_CUDA(mark(4));
  OMT_CUDA(launch_k(jpeg_rgb_kernel, dim3((unsigned)std::min(gp, cap), B), dim3(THREADS), 0, st, desc,
                    (const uint8_t*)scratch, out, status));
  OMT_CUDA(mark(5));
  if (sync_launches) *sync_launches = launches;
  if (stage_ms) {
    OMT_CUDA(cudaEventSynchronize(ev.e[5]));
    for (int i = 0; i < 5; ++i) OMT_CUDA(cudaEventElapsedTime(stage_ms + i, ev.e[i], ev.e[i + 1]));
  }
  return OMT_OK;
}

}  // namespace jdec
}  // namespace omt

using namespace omt;

extern "C" int omt_jpeg_decode_u8(const uint8_t* blob, long long blob_bytes, const omt_jpeg_desc* desc,
                                  const omt_jpeg_desc* desc_host, int B, uint8_t* scratch, long long scratch_bytes,
                                  uint8_t* out, long long out_bytes, int32_t* status, omt_stream_t stream) {
  OMT_ENTER();
  return jdec::decode(blob, blob_bytes, desc, desc_host, B, scratch, scratch_bytes, out, out_bytes, status, nullptr,
                      nullptr, stream);
}

extern "C" int omt_jpeg_decode_u8_timed(const uint8_t* blob, long long blob_bytes, const omt_jpeg_desc* desc,
                                        const omt_jpeg_desc* desc_host, int B, uint8_t* scratch, long long scratch_bytes,
                                        uint8_t* out, long long out_bytes, int32_t* status, float* stage_ms,
                                        int* sync_launches, omt_stream_t stream) {
  OMT_ENTER();
  return jdec::decode(blob, blob_bytes, desc, desc_host, B, scratch, scratch_bytes, out, out_bytes, status, stage_ms,
                      sync_launches, stream);
}
