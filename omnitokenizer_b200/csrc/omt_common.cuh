// Shared helpers for the omnitok_b200 kernels (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <atomic>
#include <initializer_list>
#include "../../include/omnitok_b200.h"

namespace omt {

// ---- host runtime (runtime.cu) ------------------------------------------------------------------------------------------
constexpr int MAX_DEVICES = 64;   // device ordinals the per-device caches cover

void set_error(const char* fmt, ...);
// OMT_OK when the current device is sm_90 (properties cached per device); it then becomes this thread's launch device,
// the one sm_count() and KernelSetup work on, until the next check.  Every entry point calls it first (OMT_ENTER).
int check_device();
int sm_count();

// A tiled TMA map over `base` with 128-byte swizzle, 256-byte L2 promotion and no out-of-bounds fill; unit element strides.
int encode_tiled(CUtensorMap* m, CUtensorMapDataType dt, const void* base, int rank, const cuuint64_t* dims,
                 const cuuint64_t* strides, const cuuint32_t* box);

// Launch setup of one kernel on each device, kept as a function-local static at its launcher (zero-initialised, so there
// is no constructor to run).  A call that finds the device already set up is one atomic load; first-time setup and
// growth take one library-wide lock and check again inside it.
class KernelSetup {
 public:
  // Raise the kernel's dynamic shared-memory limit on the launch device to at least `bytes`.
  template <typename K> int smem(K* kernel, size_t bytes) { return smem_impl(reinterpret_cast<const void*>(kernel), bytes); }
  // The same, then *ctas = the CTAs of `threads` threads resident at once on the device (occupancy x SMs).  Counted on
  // the first call per device, so a launcher passes the same `bytes` every time; a kernel no SM can hold is refused.
  template <typename K> int resident(K* kernel, int threads, size_t bytes, int* ctas) {
    return resident_impl(reinterpret_cast<const void*>(kernel), threads, bytes, ctas);
  }

 private:
  int smem_impl(const void* kernel, size_t bytes);
  int resident_impl(const void* kernel, int threads, size_t bytes, int* ctas);
  int grow(const void* kernel, int dev, size_t bytes);   // with the lock held
  std::atomic<int> smem_[MAX_DEVICES];   // the limit set on each device, 0 before the first call
  std::atomic<int> ctas_[MAX_DEVICES];   // resident CTAs on each device, 0 before the first resident()
};

#define OMT_REQUIRE(cond, ...)                  \
  do {                                          \
    if (!(cond)) {                              \
      omt::set_error(__VA_ARGS__);              \
      return OMT_E_ARG;                         \
    }                                           \
  } while (0)

#define OMT_CUDA(call)                                                            \
  do {                                                                            \
    cudaError_t e__ = (call);                                                     \
    if (e__ != cudaSuccess) {                                                     \
      omt::set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__),     \
                     __FILE__, __LINE__);                                         \
      return OMT_E_CUDA;                                                          \
    }                                                                             \
  } while (0)

// Host check of the pointers a kernel reads or writes with vector accesses: every non-NULL one is a multiple of `bytes`.
// A misaligned vector access is a device fault, so the entry points refuse such pointers before any launch.
inline bool aligned_to(size_t bytes, std::initializer_list<const void*> ptrs) {
  for (const void* p : ptrs)
    if (reinterpret_cast<uintptr_t>(p) % bytes != 0) return false;
  return true;
}

#define OMT_ENTER()                      \
  do {                                   \
    int rc__ = omt::check_device();      \
    if (rc__ != OMT_OK) return rc__;     \
  } while (0)

#define OMT_LAUNCH_CHECK() OMT_CUDA(cudaGetLastError())

// ---- programmatic dependent launch (PDL) ---------------------------------------------------------------
// Every kernel calls pdl_sync() before its first global-memory access: griddepcontrol.wait blocks until the
// previous kernel in the stream has completed and flushed (a no-op when the launch carried no PDL attribute);
// launch_dependents then lets the NEXT kernel's CTAs be scheduled as soon as all of ours are resident, so its
// prologue (barrier init, descriptor prefetch, launch latency) overlaps our last wave.
__device__ __forceinline__ void pdl_sync() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
extern int g_pdl;   // omt_set_option("pdl", 0|1)

template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = g_pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---- fp16 hi / lo operand split of the f16x3 tensor-core path -----------------------------------------------------------
// x ~= hi + lo * 2^-11 with hi = fp16(x) (round to nearest, saturating at +-65504) and lo = fp16((x - hi) * 2^11):
// 11 + 11 significant bits, representation error <= 2^-23 |x| (tighter than the tf32 hi/lo split), and both halves are
// 16-bit operands of f16 wgmma (2x the tf32 rate, half the operand bytes).  The 2^11 keeps lo in fp16's normal
// range for every |x| < 65504; the cross products  hi.lo + lo.hi  therefore carry a factor 2^11 and accumulate in their
// own fp32 accumulator, folded in as  main + cross * 2^-11  by the epilogue.
constexpr float F16X3_LO_SCALE = 2048.0f;
__device__ __forceinline__ uint32_t pack_f16x2_sat(float a, float b) {   // {low half = a, high half = b}
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}
__device__ __forceinline__ float2 unpack_f16x2(uint32_t h) {
  float2 f;
  asm("{\n\t.reg .b16 l, u;\n\tmov.b32 {l, u}, %2;\n\tcvt.f32.f16 %0, l;\n\tcvt.f32.f16 %1, u;\n\t}" : "=f"(f.x), "=f"(f.y) : "r"(h));
  return f;
}
// split two consecutive values: hi2 / lo2 are the packed 32-bit words of the two planes
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi2, uint32_t& lo2) {
  hi2 = pack_f16x2_sat(a, b);
  const float2 h = unpack_f16x2(hi2);
  lo2 = pack_f16x2_sat((a - h.x) * F16X3_LO_SCALE, (b - h.y) * F16X3_LO_SCALE);
}
// 4 consecutive values -> one 8-byte store per plane
__device__ __forceinline__ void store_split4(uint16_t* hi, uint16_t* lo, size_t off, float4 v) {
  uint2 h, l;
  split2(v.x, v.y, h.x, l.x);
  split2(v.z, v.w, h.y, l.y);
  *reinterpret_cast<uint2*>(hi + off) = h;
  *reinterpret_cast<uint2*>(lo + off) = l;
}
__device__ __forceinline__ void store_split2(uint16_t* hi, uint16_t* lo, size_t off, float2 v) {
  uint32_t h, l;
  split2(v.x, v.y, h, l);
  *reinterpret_cast<uint32_t*>(hi + off) = h;
  *reinterpret_cast<uint32_t*>(lo + off) = l;
}

// ---- row-scaled planes (single-accumulator form) ------------------------------------------------------------------------
// When a producer sees a whole row (LayerNorm, the patch gather) it can do better than the fixed 2^11: the row is
// multiplied by a power of two that puts its largest magnitude in [2^14, 2^15), hi = fp16(x'), lo = fp16(x' - hi)
// UNSCALED.  fp16 keeps 11 significant bits down to 2^-14, so every element within 2^16 of the row maximum is carried to
// 2^-23 relative and smaller ones to 2^-40 of the row maximum.  With the weights pre-scaled the same way per matrix, the
// three products hi.hi + hi.lo + lo.hi share ONE fp32 accumulator (half the accumulator registers) and the epilogue
// multiplies by the exact inverse scales.  row_scale(): scale and inverse for a row whose largest |value| is mx.
__device__ __forceinline__ void row_scale(float mx, float& scale, float& inv) {
  uint32_t eb = (__float_as_uint(mx) >> 23) & 0xffu;          // mx in [2^(eb-127), 2^(eb-126))
  eb = eb < 15u ? 15u : (eb > 254u ? 254u : eb);              // all-zero rows / inf: clamp, both factors stay normal floats
  scale = __uint_as_float((268u - eb) << 23);                 // 2^(141 - eb): row maximum -> [2^14, 2^15)
  inv = __uint_as_float((eb - 14u) << 23);                    // 2^(eb - 141)
}
__device__ __forceinline__ void split2u(float a, float b, uint32_t& hi2, uint32_t& lo2) {     // a, b already row-scaled
  hi2 = pack_f16x2_sat(a, b);
  const float2 h = unpack_f16x2(hi2);
  lo2 = pack_f16x2_sat(a - h.x, b - h.y);
}
__device__ __forceinline__ void store_split4u(uint16_t* hi, uint16_t* lo, size_t off, float4 v, float scale) {
  uint2 h, l;
  split2u(v.x * scale, v.y * scale, h.x, l.x);
  split2u(v.z * scale, v.w * scale, h.y, l.y);
  *reinterpret_cast<uint2*>(hi + off) = h;
  *reinterpret_cast<uint2*>(lo + off) = l;
}
// fp32 pairs: two scalar ops per call (sm_90 has no packed f32x2 arithmetic); each half rounds like the scalar op
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float ex2_fast(float x) {      // MUFU.EX2 alone; results below 2^-126 flush to zero
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// unscaled hi / lo planes of a pair (the pair already carries its row scale)
__device__ __forceinline__ void split2u_pk(float2 v, uint32_t& hi2, uint32_t& lo2) {
  hi2 = pack_f16x2_sat(v.x, v.y);
  const float2 d = ffma2(unpack_f16x2(hi2), make_float2(-1.f, -1.f), v);      // v - hi, exact
  lo2 = pack_f16x2_sat(d.x, d.y);
}
// 8 consecutive row-scaled values -> one 16-byte store per plane
__device__ __forceinline__ void store_split8u(uint16_t* hi, uint16_t* lo, size_t off, float4 a, float4 b, float scale) {
  uint4 h, l;
  split2u(a.x * scale, a.y * scale, h.x, l.x);
  split2u(a.z * scale, a.w * scale, h.y, l.y);
  split2u(b.x * scale, b.y * scale, h.z, l.z);
  split2u(b.z * scale, b.w * scale, h.w, l.w);
  *reinterpret_cast<uint4*>(hi + off) = h;
  *reinterpret_cast<uint4*>(lo + off) = l;
}
__device__ __forceinline__ float max4abs(float4 v) { return fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))); }

__device__ __forceinline__ float gelu_erf(float x) {
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}

// ---- packed batches (include/omnitok_b200.h, "varlen" entry points) ----------------------------------------------------
// Sample b owns latent frames [t_off[b], t_off[b+1]) and canonical rows [t_off[b] * N, t_off[b+1] * N).  The host copy of
// the table is checked before any launch: t_off[0] == 0, every sample 1..17 frames long, t_off[B] * N == M rows.
// *t_max receives the longest sample.
inline int check_t_off(const char* who, const int32_t* t_off_host, const int32_t* t_off, int B, long long M, long long N,
                       int* t_max) {
  OMT_REQUIRE(t_off_host && t_off, "%s: null layout table", who);
  OMT_REQUIRE(B >= 0 && B <= 65535, "%s: B=%d samples unsupported (0..65535)", who, B);
  OMT_REQUIRE(t_off_host[0] == 0, "%s: t_off[0]=%d must be 0", who, t_off_host[0]);
  int mx = 0;
  for (int b = 0; b < B; ++b) {
    const int tb = t_off_host[b + 1] - t_off_host[b];
    OMT_REQUIRE(tb >= 1 && tb <= 17, "%s: sample %d has T'=%d latent frames (t_off must increase by 1..17)", who, b, tb);
    mx = tb > mx ? tb : mx;
  }
  OMT_REQUIRE((long long)t_off_host[B] * N == M, "%s: t_off[B]=%d frames of %lld rows != %lld rows", who, t_off_host[B], N, M);
  *t_max = mx;
  return OMT_OK;
}

// logical GEMM row -> physical row (see include/omnitok_b200.h)
__host__ __device__ __forceinline__ long long map_row(int r, int seg, int seg_stride, int seg_off) {
  if (seg <= 0) return r;
  return (long long)(r / seg) * seg_stride + seg_off + (r % seg);
}

struct GemmArgs {
  const float* A; int lda; int a_seg, a_seg_stride, a_seg_off;
  const float* W;
  float* C; int ldc; int c_seg, c_seg_stride, c_seg_off;
  int M, N, K;
  const float* bias; const float* residual; int ldr;
  const float* A2; int n_split;   // dual-A form: output columns >= n_split are computed from A2 (same lda / row map)
  // OMT_EPI_QKV: heads (64 columns) below qk_cols get rope + l2norm + per-dim scale in the epilogue
  const float* rope_cos; const float* rope_sin; const float* q_scale; const float* k_scale;
  int qk_cols; int tokens;        // rope position of row m is m % tokens; columns < qk_cols/2 use q_scale, the rest k_scale
};

}  // namespace omt
