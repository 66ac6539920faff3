// Codebook path: pre_vq projection (+l2 normalise) and the exact-fp32 nearest-neighbour search with the
// reference's  (sum z^2 - 2 z.E) + sum E^2  association and first-min tie rule -- fused into one cluster
// kernel (vq_fused_kernel) -- and the decode-side gather + post_vq projection.
#include "omt_common.cuh"
#include "tc_ptx.cuh"

namespace omt {

// ---------------------------------------------------------------------------------------
// pre_vq: z[M, CD] = x[M, C] . W[CD, C]^T + b   (C = 512 -> 4 float4 per lane), optional l2 norm.
// One warp per row; W staged in shared memory.
// ---------------------------------------------------------------------------------------
template <int CD>
__global__ void __launch_bounds__(256) pre_vq_kernel(const float* __restrict__ x, int ldx,
                                                     const float* __restrict__ Wt,
                                                     const float* __restrict__ b,
                                                     float* __restrict__ z, int M, int C, int l2) {
  pdl_sync();
  extern __shared__ float4 wsm4[];   // [CD][C/4]
  const int C4 = C >> 2;
  for (int i = threadIdx.x; i < CD * C4; i += blockDim.x) wsm4[i] = reinterpret_cast<const float4*>(Wt)[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warps = blockDim.x >> 5;
  for (int row = blockIdx.x * warps + (threadIdx.x >> 5); row < M; row += gridDim.x * warps) {
    const float4* xr = reinterpret_cast<const float4*>(x + (size_t)row * ldx);
    float acc[CD];
#pragma unroll
    for (int j = 0; j < CD; ++j) acc[j] = 0.f;
    for (int c = lane; c < C4; c += 32) {
      const float4 xv = xr[c];
#pragma unroll
      for (int j = 0; j < CD; ++j) {
        const float4 wv = wsm4[j * C4 + c];
        acc[j] = fmaf(xv.x, wv.x, acc[j]);
        acc[j] = fmaf(xv.y, wv.y, acc[j]);
        acc[j] = fmaf(xv.z, wv.z, acc[j]);
        acc[j] = fmaf(xv.w, wv.w, acc[j]);
      }
    }
    float ss = 0.f;
#pragma unroll
    for (int j = 0; j < CD; ++j) {
      acc[j] = warp_sum(acc[j]) + b[j];
      ss = fmaf(acc[j], acc[j], ss);
    }
    float den = 1.f;
    if (l2) den = fmaxf(sqrtf(ss), 1e-12f);
    if (lane == 0) {
#pragma unroll
      for (int j = 0; j < CD; ++j) z[(size_t)row * CD + j] = l2 ? acc[j] / den : acc[j];
    }
  }
}

// ---------------------------------------------------------------------------------------
// Fused VQ lookup: pre_vq projection + l2 normalise + || z ||^2 - 2 z E^T + || E ||^2 + argmin (+ usage histogram) in
// ONE launch (modules/codebook.py:82-86 after omnitokenizer.py:248-252).
//
// A cluster of 8 CTAs owns a block of 128 R rows (R = 4, or 2 for small inputs); CTA r of the cluster
//   A. projects rows [16 R r, 16 R (r + 1)) of the block (warp per row, the arithmetic of pre_vq_kernel) and broadcasts
//      the 8 floats of each z row into the z table of ALL 8 CTAs through distributed shared memory (and to global z);
//   B. searches ALL rows of the block against ITS slice of the codebook (n_codes / 8 codes + their || E ||^2, staged
//      once in shared memory with coalesced 16-byte reads): a thread keeps R rows of z in registers, so one broadcast
//      read of a code (36 bytes) feeds 8 R FMAs.  The minimum is tracked per GROUP of 8 codes (one FMNMX per distance,
//      one compare-and-select per group instead of per code -- the per-code compare / select pair was a third of the
//      old kernel's instructions); the winning group is re-evaluated once at the end with the same instruction
//      sequence, so the first code whose distance equals the group minimum bit for bit is the first minimum;
//   C. sends its per-row (distance, index) to the CTA that owns the row (DSMEM again); the owner takes the first minimum
//      over the 8 slices in ascending slice order == torch.argmin's first-min rule, writes the int64 index and bumps
//      the histogram that replaces torch.unique (codebook.py:65).
// Distances keep the reference association (sum z^2 - 2 z.E) + sum E^2 with a sequential fma chain over the 8 dims.
// Shared memory: [slice 36 B / code | projection weights during A]  [z table, reused for the partial minima in C].
// ---------------------------------------------------------------------------------------
constexpr int VQF_SLICES = 8;                 // cluster size = codebook slices
constexpr int VQF_THREADS = 128;
constexpr int VQF_GROUP = 8;                  // codes per minimum group

// bytes of the first shared-memory region: the table slice (36 B / code), or the projection weights of phase A if those
// are larger (small codebooks); the z table starts right after it
__host__ __device__ __forceinline__ size_t vq_region0_bytes(int per, bool project, int C) {
  const size_t table = (size_t)per * 36, weights = project ? (size_t)32 * C : 0;
  return table > weights ? table : weights;
}

// distance of one row (2 z in z2[], sum z^2 in zz) to one code: the exact instruction sequence both passes share
__device__ __forceinline__ float vq_dist(const float (&z2)[8], float zz, const float4 ea, const float4 eb, float ek) {
  float dot = __fmul_rn(z2[0], ea.x);
  dot = fmaf(z2[1], ea.y, dot); dot = fmaf(z2[2], ea.z, dot); dot = fmaf(z2[3], ea.w, dot);
  dot = fmaf(z2[4], eb.x, dot); dot = fmaf(z2[5], eb.y, dot); dot = fmaf(z2[6], eb.z, dot); dot = fmaf(z2[7], eb.w, dot);
  return __fadd_rn(__fsub_rn(zz, dot), ek);
}

template <bool PROJECT, int R>       // PROJECT: rows come from x . Wt^T + b (fused pre_vq); else z is given.  R rows / thread
__global__ void __cluster_dims__(VQF_SLICES, 1, 1) __launch_bounds__(VQF_THREADS)
vq_fused_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ Wt, const float* __restrict__ bias, int C, int l2,
                const float* __restrict__ z_in, float* __restrict__ z_out, const float* __restrict__ E,
                const float* __restrict__ e2, int M, int n_codes, int64_t* __restrict__ idx, int32_t* __restrict__ counts) {
  constexpr int ROWS = R * VQF_THREADS;        // rows per cluster
  constexpr int OWN = ROWS / VQF_SLICES;       // rows projected / finalised per CTA
  pdl_sync();
  extern __shared__ __align__(16) uint8_t vq_smem[];
  const int per = n_codes / VQF_SLICES;
  float4* esm = reinterpret_cast<float4*>(vq_smem);                          // [per][2] float4: this slice of the table
  float* e2s = reinterpret_cast<float*>(esm + 2 * per);                      // [per]
  float4* wsm = reinterpret_cast<float4*>(vq_smem);                          // PROJECT, phase A only: [8][C/4] weights
  float4* zsm = reinterpret_cast<float4*>(vq_smem + vq_region0_bytes(per, PROJECT, C));   // [ROWS][2] float4: the block's z rows
  float2* part = reinterpret_cast<float2*>(zsm);                             // phase C: [8 slices][OWN] (distance, index bits)
  const uint32_t rank = ptx::cluster_ctarank();
  const int row0 = (blockIdx.x / VQF_SLICES) * ROWS;
  const int k0 = (int)rank * per;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  ptx::cluster_arrive();          // no CTA touches a peer's shared memory before every CTA of the cluster is running

  // ---- A. this CTA's OWN rows of z -> the z table of every CTA of the cluster
  const uint32_t zsm_s = static_cast<uint32_t>(__cvta_generic_to_shared(zsm));
  if (PROJECT) {
    const int C4 = C >> 2;
    for (int i = tid; i < 8 * C4; i += VQF_THREADS) wsm[i] = reinterpret_cast<const float4*>(Wt)[i];
    __syncthreads();
    ptx::cluster_wait();
    for (int rr = warp; rr < OWN; rr += VQF_THREADS / 32) {
      const int lrow = (int)rank * OWN + rr, row = row0 + lrow;
      float acc[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = 0.f;
      if (row < M) {
        const float4* xr = reinterpret_cast<const float4*>(x + (size_t)row * ldx);
        for (int c = lane; c < C4; c += 32) {
          const float4 xv = xr[c];
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float4 wv = wsm[j * C4 + c];
            acc[j] = fmaf(xv.x, wv.x, acc[j]);
            acc[j] = fmaf(xv.y, wv.y, acc[j]);
            acc[j] = fmaf(xv.z, wv.z, acc[j]);
            acc[j] = fmaf(xv.w, wv.w, acc[j]);
          }
        }
      }
      float ss = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        acc[j] = warp_sum(acc[j]) + bias[j];
        ss = fmaf(acc[j], acc[j], ss);
      }
      const float den = l2 ? fmaxf(sqrtf(ss), 1e-12f) : 1.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = l2 ? acc[j] / den : acc[j];
      if (row >= M) {
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.f;
      }
      if (lane < VQF_SLICES) {            // lane r writes the row into CTA r's table
        const uint32_t dst = ptx::mapa(zsm_s + (uint32_t)lrow * 32u, (uint32_t)lane);
        asm volatile("st.shared::cluster.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(dst), "f"(acc[0]), "f"(acc[1]), "f"(acc[2]), "f"(acc[3]) : "memory");
        asm volatile("st.shared::cluster.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(dst + 16u), "f"(acc[4]), "f"(acc[5]), "f"(acc[6]), "f"(acc[7]) : "memory");
      }
      if (lane == 0 && row < M && z_out != nullptr) {
        float4* zo = reinterpret_cast<float4*>(z_out + (size_t)row * 8);
        zo[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
        zo[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
      }
    }
  } else {
    ptx::cluster_wait();
    for (int i = tid; i < OWN * 2; i += VQF_THREADS) {              // this CTA's rows, 2 float4 each
      const int lrow = (int)rank * OWN + (i >> 1), row = row0 + lrow;
      const float4 v = row < M ? reinterpret_cast<const float4*>(z_in + (size_t)row * 8)[i & 1] : make_float4(0.f, 0.f, 0.f, 0.f);
      for (uint32_t r = 0; r < VQF_SLICES; ++r) {
        const uint32_t dst = ptx::mapa(zsm_s + (uint32_t)lrow * 32u + (uint32_t)(i & 1) * 16u, r);
        asm volatile("st.shared::cluster.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(dst), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
      }
    }
  }
  ptx::cluster_arrive();          // every CTA holds all z rows after this barrier; this CTA is also done with wsm
  ptx::cluster_wait();
  for (int i = tid; i < 2 * per; i += VQF_THREADS) esm[i] = reinterpret_cast<const float4*>(E + (size_t)k0 * 8)[i];
  for (int i = tid; i < per; i += VQF_THREADS) e2s[i] = e2[k0 + i];

  // ---- B. R rows per thread (rows tid + 128 r) against this CTA's slice
  float z2[R][8];            // 2 * z: (2 * z) @ E^T, the factor 2 is exact
  float zz[R];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const float4 za = zsm[2 * (tid + r * VQF_THREADS)], zb = zsm[2 * (tid + r * VQF_THREADS) + 1];
    // sum z^2 exactly as torch's (z**2).sum(dim=1): sequential over the 8 channels
    float s = za.x * za.x;
    s += za.y * za.y; s += za.z * za.z; s += za.w * za.w;
    s += zb.x * zb.x; s += zb.y * zb.y; s += zb.z * zb.z; s += zb.w * zb.w;
    zz[r] = s;
    z2[r][0] = 2.f * za.x; z2[r][1] = 2.f * za.y; z2[r][2] = 2.f * za.z; z2[r][3] = 2.f * za.w;
    z2[r][4] = 2.f * zb.x; z2[r][5] = 2.f * zb.y; z2[r][6] = 2.f * zb.z; z2[r][7] = 2.f * zb.w;
  }
  ptx::cluster_arrive();          // this CTA's z table is dead: the peers may overwrite it with partial minima (phase C)
  __syncthreads();              // the table slice is staged
  float best[R];
  int bg[R];
#pragma unroll
  for (int r = 0; r < R; ++r) { best[r] = INFINITY; bg[r] = 0; }
  for (int g = 0; g < per; g += VQF_GROUP) {
    float gm[R];
#pragma unroll
    for (int r = 0; r < R; ++r) gm[r] = INFINITY;
#pragma unroll
    for (int c = 0; c < VQF_GROUP; ++c) {
      const float4 ea = esm[2 * (g + c)], eb = esm[2 * (g + c) + 1];
      const float ek = e2s[g + c];
#pragma unroll
      for (int r = 0; r < R; ++r) gm[r] = fminf(gm[r], vq_dist(z2[r], zz[r], ea, eb, ek));
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
      if (gm[r] < best[r]) { best[r] = gm[r]; bg[r] = g; }          // strict <  => the first group holding the minimum
    }
  }
  // the winning group once more: the first code whose distance equals the minimum bit for bit
  int bi[R];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    bi[r] = bg[r];
    bool found = false;
#pragma unroll
    for (int c = 0; c < VQF_GROUP; ++c) {
      const float d = vq_dist(z2[r], zz[r], esm[2 * (bg[r] + c)], esm[2 * (bg[r] + c) + 1], e2s[bg[r] + c]);
      if (!found && d == best[r]) { bi[r] = bg[r] + c; found = true; }
    }
  }
  // ---- C. partial minima -> the owner CTA of each row (every CTA has left its z table: second cluster barrier)
  ptx::cluster_wait();
  const uint32_t part_s = static_cast<uint32_t>(__cvta_generic_to_shared(part));
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int lrow = tid + r * VQF_THREADS;
    const uint32_t owner = (uint32_t)(lrow / OWN);
    const uint32_t dst = ptx::mapa(part_s + (uint32_t)((rank * OWN + (lrow % OWN)) * 8), owner);
    asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(dst), "f"(best[r]), "f"(__int_as_float(k0 + bi[r])) : "memory");
  }
  ptx::cluster_arrive();
  ptx::cluster_wait();
  if (tid < OWN) {
    const int row = row0 + (int)rank * OWN + tid;
    if (row < M) {
      float2 b0 = part[tid];
#pragma unroll
      for (int s = 1; s < VQF_SLICES; ++s) {
        const float2 c = part[s * OWN + tid];
        if (c.x < b0.x) b0 = c;                 // ascending slices, strict <: the first minimum over the whole codebook
      }
      const int code = __float_as_int(b0.y);
      idx[row] = code;
      if (counts != nullptr) atomicAdd(counts + code, 1);
    }
  }
}

// ---------------------------------------------------------------------------------------
// post_vq: X[M, C] = zrow[M, CD] . W[C, CD]^T + b, zrow = E[idx] | zc | (E[idx]-z)+z.
// Block = C/4 threads rounded up to 128 (C <= 512) or 256 (C <= 1024, the wide kernel); a thread owns 4 output channels
// (its 4 x CD weights live in registers).  Both kernels run the same body: only the launch bounds differ.
// ---------------------------------------------------------------------------------------
constexpr int POSTVQ_ROWS = 32;

template <int CD>
__device__ __forceinline__ void post_vq_rows(const int64_t* __restrict__ idx, const float* __restrict__ E,
                                             const float* __restrict__ zc, const float* __restrict__ zst,
                                             float* __restrict__ zq_out, const float* __restrict__ Wt,
                                             const float* __restrict__ b, float* __restrict__ X, int M, int C) {
  __shared__ float rows[POSTVQ_ROWS][CD];
  const int r0 = blockIdx.x * POSTVQ_ROWS;
  for (int i = threadIdx.x; i < POSTVQ_ROWS * CD; i += blockDim.x) {
    const int r = r0 + i / CD, j = i % CD;
    float v = 0.f;
    if (r < M) {
      if (idx != nullptr) {
        v = E[(size_t)idx[r] * CD + j];
        if (zst != nullptr) {                       // straight-through rounding (codebook.py:120)
          const float zz = zst[(size_t)r * CD + j];
          v = (v - zz) + zz;
        }
      } else {
        v = zc[(size_t)r * CD + j];
      }
      if (zq_out != nullptr) zq_out[(size_t)r * CD + j] = v;
    }
    rows[i / CD][j] = v;
  }
  __syncthreads();
  const int c = threadIdx.x * 4;
  if (c >= C) return;
  float w[4][CD];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < CD; ++j) w[i][j] = Wt[(size_t)(c + i) * CD + j];
  const float4 bb = *reinterpret_cast<const float4*>(b + c);
  for (int rr = 0; rr < POSTVQ_ROWS; ++rr) {
    const int r = r0 + rr;
    if (r >= M) break;
    float o[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int j = 0; j < CD; ++j) {
      const float zv = rows[rr][j];
#pragma unroll
      for (int i = 0; i < 4; ++i) o[i] = fmaf(zv, w[i][j], o[i]);
    }
    *reinterpret_cast<float4*>(X + (size_t)r * C + c) =
        make_float4(o[0] + bb.x, o[1] + bb.y, o[2] + bb.z, o[3] + bb.w);
  }
}

template <int CD>
__global__ void __launch_bounds__(128) post_vq_kernel(const int64_t* __restrict__ idx,
                                                      const float* __restrict__ E,
                                                      const float* __restrict__ zc,
                                                      const float* __restrict__ zst,
                                                      float* __restrict__ zq_out,
                                                      const float* __restrict__ Wt,
                                                      const float* __restrict__ b,
                                                      float* __restrict__ X, int M, int C) {
  pdl_sync();
  post_vq_rows<CD>(idx, E, zc, zst, zq_out, Wt, b, X, M, C);
}

// C in (512, 1024]: 256 threads
template <int CD>
__global__ void __launch_bounds__(256) post_vq_wide_kernel(const int64_t* __restrict__ idx,
                                                           const float* __restrict__ E,
                                                           const float* __restrict__ zc,
                                                           const float* __restrict__ zst,
                                                           float* __restrict__ zq_out,
                                                           const float* __restrict__ Wt,
                                                           const float* __restrict__ b,
                                                           float* __restrict__ X, int M, int C) {
  pdl_sync();
  post_vq_rows<CD>(idx, E, zc, zst, zq_out, Wt, b, X, M, C);
}

}  // namespace omt

using namespace omt;

extern "C" int omt_pre_vq(const float* x, int ldx, const float* Wt, const float* b, float* z, int M, int C,
                          int cd, int l2, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(x && Wt && b && z, "omt_pre_vq: null pointer");
  OMT_REQUIRE(C % 4 == 0 && ldx % 4 == 0 && C <= 1024, "omt_pre_vq: bad C/ldx");
  OMT_REQUIRE(aligned_to(16, {x, Wt}), "omt_pre_vq: x and Wt must be 16-byte aligned");
  OMT_REQUIRE(cd == 8 || cd == 16, "omt_pre_vq: codebook_dim %d unsupported (8 or 16)", cd);
  if (M == 0) return OMT_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t smem = (size_t)cd * C * sizeof(float);
  int blocks = (M + 7) / 8;
  const int cap = omt::sm_count() * 4;
  if (blocks > cap) blocks = cap;
  if (cd == 8) {
    OMT_CUDA(launch_k(pre_vq_kernel<8>, dim3(blocks), dim3(256), smem, st, x, ldx, Wt, b, z, M, C, l2));
  } else {
    static KernelSetup setup;
    const int rc = setup.smem(pre_vq_kernel<16>, 16 * 1024 * 4);   // the widest row (C = 1024) once
    if (rc != OMT_OK) return rc;
    OMT_CUDA(launch_k(pre_vq_kernel<16>, dim3(blocks), dim3(256), smem, st, x, ldx, Wt, b, z, M, C, l2));
  }
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

template <bool PROJECT, int R>
static int vq_launch_r(const float* x, int ldx, const float* Wt, const float* b, int C, int l2, const float* z_in, float* z_out,
                       const float* E, const float* e2, int M, int n_codes, int64_t* idx, int32_t* counts, cudaStream_t st) {
  const int per = n_codes / VQF_SLICES;
  const size_t smem = vq_region0_bytes(per, PROJECT, C) + (size_t)R * VQF_THREADS * 32;
  OMT_REQUIRE(smem <= 200 * 1024, "omt_vq: n_codes=%d too large for the shared-memory table slice (C=%d, %d rows per thread)",
              n_codes, C, R);
  static KernelSetup setup;
  const int rc = setup.smem(vq_fused_kernel<PROJECT, R>, smem);
  if (rc != OMT_OK) return rc;
  const int rows = R * VQF_THREADS;
  const unsigned blocks = (unsigned)((M + rows - 1) / rows) * VQF_SLICES;
  OMT_CUDA(launch_k(vq_fused_kernel<PROJECT, R>, dim3(blocks), dim3(VQF_THREADS), smem, st, x, ldx, Wt, b, C, l2, z_in, z_out, E, e2,
                    M, n_codes, idx, counts));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}

static int vq_launch(bool project, const float* x, int ldx, const float* Wt, const float* b, int C, int l2, const float* z_in,
                     float* z_out, const float* E, const float* e2, int M, int n_codes, int64_t* idx, int32_t* counts,
                     cudaStream_t st) {
  OMT_REQUIRE(n_codes % (VQF_SLICES * VQF_GROUP) == 0 && n_codes >= VQF_SLICES * VQF_GROUP, "omt_vq: n_codes=%d is not a positive multiple of 64", n_codes);
  // 4 rows per thread amortise the table reads best; small inputs take 2 so that more SMs get a cluster
  const bool small = (M + 4 * VQF_THREADS - 1) / (4 * VQF_THREADS) * VQF_SLICES < omt::sm_count();
  if (project)
    return small ? vq_launch_r<true, 2>(x, ldx, Wt, b, C, l2, z_in, z_out, E, e2, M, n_codes, idx, counts, st)
                 : vq_launch_r<true, 4>(x, ldx, Wt, b, C, l2, z_in, z_out, E, e2, M, n_codes, idx, counts, st);
  return small ? vq_launch_r<false, 2>(x, ldx, Wt, b, C, l2, z_in, z_out, E, e2, M, n_codes, idx, counts, st)
               : vq_launch_r<false, 4>(x, ldx, Wt, b, C, l2, z_in, z_out, E, e2, M, n_codes, idx, counts, st);
}

extern "C" int omt_vq_search(const float* z, const float* E, const float* e2, int M, int n_codes,
                             int64_t* idx, int32_t* counts, omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(z && E && e2 && idx, "omt_vq_search: null pointer");
  OMT_REQUIRE(aligned_to(16, {z, E}), "omt_vq_search: z and E must be 16-byte aligned");
  if (M == 0) return OMT_OK;
  return vq_launch(false, nullptr, 0, nullptr, nullptr, 0, 0, z, nullptr, E, e2, M, n_codes, idx, counts, (cudaStream_t)stream);
}

extern "C" int omt_vq_fused(const float* x, int ldx, const float* Wt, const float* b, int C, int l2, float* z,
                            const float* E, const float* e2, int M, int n_codes, int64_t* idx, int32_t* counts,
                            omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(x && Wt && b && E && e2 && idx, "omt_vq_fused: null pointer");
  OMT_REQUIRE(C % 4 == 0 && ldx % 4 == 0 && C <= 1024, "omt_vq_fused: bad C/ldx");
  OMT_REQUIRE(aligned_to(16, {x, Wt, z, E}), "omt_vq_fused: x, Wt, z and E must be 16-byte aligned");
  if (M == 0) return OMT_OK;
  return vq_launch(true, x, ldx, Wt, b, C, l2, nullptr, z, E, e2, M, n_codes, idx, counts, (cudaStream_t)stream);
}

extern "C" int omt_post_vq(const int64_t* idx, const float* E, const float* zc, const float* z_st_from,
                           float* zq_out, const float* Wt, const float* b, float* X, int M, int C, int cd,
                           omt_stream_t stream) {
  OMT_ENTER();
  OMT_REQUIRE(Wt && b && X, "omt_post_vq: null pointer");
  OMT_REQUIRE((idx != nullptr && E != nullptr) || zc != nullptr, "omt_post_vq: need idx+E or zc");
  OMT_REQUIRE(C % 4 == 0 && C <= 1024, "omt_post_vq: C=%d unsupported (C %% 4 == 0, C <= 1024)", C);
  OMT_REQUIRE(aligned_to(16, {X, b}), "omt_post_vq: X and b must be 16-byte aligned");
  OMT_REQUIRE(cd == 8, "omt_post_vq: codebook_dim %d unsupported (8)", cd);
  if (M == 0) return OMT_OK;
  const dim3 grid((M + POSTVQ_ROWS - 1) / POSTVQ_ROWS);
  if (C <= 512)
    OMT_CUDA(launch_k(post_vq_kernel<8>, grid, dim3(128), 0, (cudaStream_t)stream, idx, E, zc, z_st_from, zq_out, Wt, b, X, M, C));
  else
    OMT_CUDA(launch_k(post_vq_wide_kernel<8>, grid, dim3(256), 0, (cudaStream_t)stream, idx, E, zc, z_st_from, zq_out, Wt, b, X, M, C));
  OMT_LAUNCH_CHECK();
  return OMT_OK;
}
