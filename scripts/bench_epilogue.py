"""Epilogue cost of the plane-writing f16x3 GEMMs, separated from their mainloop (CUDA events, L2 flushed, median of
7 launches):
   python scripts/bench_epilogue.py [--rounds R] [--M M]

At M = 40 960 it times, on the row-scaled ping-pong kernel:
  * FF1 + GEGLU -> U planes (N 2 816, K 512) and dual-A QKV -> planes (rope, l2 norm, scales, v split; N 1 536, K 512)
    as the library builds them;
  * the same kernel with its epilogue replaced by a plain store of the same bytes: "store-only".  That variant is built
    here, into a scratch library in a temporary directory, from the tree's gemm_wgmma.cuh: it keeps the mainloop, the
    ping-pong order and the row-scale multiply, and writes each 64-column head's fragments as fp16 pairs to the hi / lo
    planes (and, for QKV, one vinv word per row and v head), 4 bytes a lane per store, as the QKV epilogue stores;
  * the plain qkv -> fp32 GEMM (N 1 536, K 512), the same mainloop with the lightest in-tree epilogue.
Each line gives the launch time and the time per tile of a CTA's walk (tiles / resident CTAs, rounded up); the gap of
the in-tree kernel to its store-only twin is what its epilogue costs beyond storing its bytes."""
import argparse
import ctypes
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from omnitokenizer_b200 import _cabi, layout as L  # noqa: E402

CSRC = os.path.join(ROOT, "omnitokenizer_b200", "csrc")

# The store-only epilogues, as full specialisations of wgg::epilogue for two epilogue numbers the library never uses,
# and a launcher that builds the tensor maps and argument block as omt_linear_h does (row-scaled form, no row maps).
SCRATCH_CU = r'''
#include "gemm_wgmma.cuh"
namespace omt {
int g_pdl = 0;
void set_error(const char* fmt, ...) { va_list ap; va_start(ap, fmt); vfprintf(stderr, fmt, ap); va_end(ap); fputc('\n', stderr); }
namespace wgg {
constexpr int STORE_U = 100, STORE_QKV = 101;

template <int EPI>
__device__ __forceinline__ void store_only(const Args& g, const float (&acc)[BN / 2], int m0, int n0, bool second, int half,
                                           int warp, int lane) {
  const int qd = lane & 3;
  int mrow[2];
  mrow[0] = m0 + half * 64 + (warp & 3) * 16 + (lane >> 2);
  mrow[1] = mrow[0] + 8;
  float v[2][BN / 4];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float* rs = second ? g.a2_rs : g.a_rs;
    const int m = mrow[h];
    const float os = g.w_scale * (m < g.M ? __ldg(rs + m) : 1.0f);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      v[h][2 * j] = acc[4 * j + 2 * h] * os;
      v[h][2 * j + 1] = acc[4 * j + 2 * h + 1] * os;
    }
  }
#pragma unroll
  for (int hd = 0; hd < BN / 64; ++hd) {
    const int nh = n0 + hd * 64;
    if (nh >= g.N) break;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = mrow[h];
      if (m >= g.M) continue;
      const float* x = &v[h][hd * 16];
      if (EPI == STORE_U) {
        // the tile's 64 U columns: head hd's fragments go to the hi plane (hd 0) or the lo plane (hd 1)
        uint16_t* p = (hd == 0 ? g.u_hi : g.u_lo) + (size_t)m * g.ldu + (n0 >> 1) + 2 * qd;
#pragma unroll
        for (int j = 0; j < 8; ++j) *reinterpret_cast<uint32_t*>(p + 8 * j) = pack_f16x2_sat(x[2 * j], x[2 * j + 1]);
      } else {
        const size_t off = (size_t)m * g.ldu + nh + 2 * qd;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          *reinterpret_cast<uint32_t*>(g.u_hi + off + 8 * j) = pack_f16x2_sat(x[2 * j], x[2 * j + 1]);
          *reinterpret_cast<uint32_t*>(g.u_lo + off + 8 * j) = pack_f16x2_sat(x[2 * j + 1], x[2 * j]);
        }
        if (nh >= g.qk_cols && qd == 0) g.vinv[(size_t)((nh - g.qk_cols) >> 6) * g.M + m] = x[0];
      }
    }
  }
}
template <>
__device__ __forceinline__ void epilogue<false, 1, STORE_U, false>(const Args& g, const float (&acc)[BN / 2], const float (&)[1],
    int m0, int n0, bool second, int half, int warp, int lane, uint8_t*, int, const CUtensorMap*, const CUtensorMap*) {
  store_only<STORE_U>(g, acc, m0, n0, second, half, warp, lane);
}
template <>
__device__ __forceinline__ void epilogue<false, 1, STORE_QKV, false>(const Args& g, const float (&acc)[BN / 2], const float (&)[1],
    int m0, int n0, bool second, int half, int warp, int lane, uint8_t*, int, const CUtensorMap*, const CUtensorMap*) {
  store_only<STORE_QKV>(g, acc, m0, n0, second, half, warp, lane);
}
}  // namespace wgg
}  // namespace omt

extern "C" int bench_store_only(const omt_linear_h_args* a, int qkv, omt_stream_t stream) {
  using namespace omt;
  using namespace omt::wgg;
  const int n_pad = (a->N + 255) / 256 * 256;
  const CUtensorMapDataType f16 = CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const bool dual = a->a2_hi != nullptr;
  CUtensorMap maps[6];
  int rc;
  if ((rc = row_map(&maps[0], f16, 2, a->a_hi, a->lda, a->M, a->K, 0, 0, 0))) return rc;
  if ((rc = row_map(&maps[1], f16, 2, a->a_lo, a->lda, a->M, a->K, 0, 0, 0))) return rc;
  if ((rc = row_map(&maps[2], f16, 2, dual ? a->a2_hi : a->a_hi, a->lda, a->M, a->K, 0, 0, 0))) return rc;
  if ((rc = row_map(&maps[3], f16, 2, dual ? a->a2_lo : a->a_lo, a->lda, a->M, a->K, 0, 0, 0))) return rc;
  if ((rc = w_map(&maps[4], f16, 2, a->w_hi, n_pad, a->K))) return rc;
  if ((rc = w_map(&maps[5], f16, 2, a->w_lo, n_pad, a->K))) return rc;
  Args g{};
  g.M = a->M; g.N = a->N; g.K = a->K;
  g.num_m_blk = (a->M + BM - 1) / BM;
  g.n_split = dual ? a->n_split : 0x7fffffff;
  g.a_rs = a->a_rs; g.a2_rs = dual ? a->a2_rs : a->a_rs; g.w_scale = a->w_scale;
  g.u_hi = a->u_hi; g.u_lo = a->u_lo; g.ldu = a->ldu;
  g.qk_cols = qkv ? a->qk_cols : 0x7fffffff; g.vinv = a->vinv;
  return qkv ? launch<false, 1, STORE_QKV>(maps, g, (cudaStream_t)stream)
             : launch<false, 1, STORE_U>(maps, g, (cudaStream_t)stream);
}
'''


def build_scratch(tmp):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    src = os.path.join(tmp, "store_only.cu")
    out = os.path.join(tmp, "libstore_only.so")
    with open(src, "w") as f:
        f.write(SCRATCH_CU)
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-shared",
                    "-Xcompiler", "-fPIC", "-I", CSRC, "-o", out, src], check=True)
    lib = ctypes.CDLL(out)
    lib.bench_store_only.restype = ctypes.c_int
    lib.bench_store_only.argtypes = [ctypes.POINTER(_cabi.LinearHArgs), ctypes.c_int, ctypes.c_void_p]
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--M", type=int, default=40960)
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds over the kernels")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_epilogue.py measures on a GPU"
    dev = torch.device("cuda:0")
    props = torch.cuda.get_device_properties(dev)
    print(f"device: {props.name}, {props.multi_processor_count} SMs", flush=True)
    tmp = tempfile.mkdtemp(prefix="omt_bench_epilogue_")
    try:
        scratch = build_scratch(tmp)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)    # the library stays mapped
    _cabi.load()

    M, C, INNER, HEADS = args.M, 512, 1365, 8
    g = torch.Generator(device=dev).manual_seed(1)
    flush = torch.zeros(64 * 1024 * 1024, device=dev)

    def timeit(fn, reps=7):
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
        for i in range(reps + 2):
            flush.add_(1.0)
            if i >= 2: evs[i - 2][0].record()
            fn()
            if i >= 2: evs[i - 2][1].record()
        torch.cuda.synchronize()
        return sorted(a.elapsed_time(b) for a, b in evs)[reps // 2] * 1e3

    def operands(N, K, dual):
        W = torch.rand(N, K, device=dev, generator=g) * 0.1 - 0.05
        A = torch.rand(M, K, device=dev, generator=g) - 0.5
        ah, al, ars = L.split_rows_rs(A)
        wh, wl, wsc = L.split_f16_rs(L.pad_rows(W, 256))
        kw = dict(a_hi=ah, a_lo=al, a_rs=ars, w_scale=wsc, w_hi=wh, w_lo=wl, lda=K, M=M, N=N, K=K)
        if dual:
            a2h, a2l, a2rs = L.split_rows_rs(A.flip(1))
            kw.update(a2_hi=a2h, a2_lo=a2l, a2_rs=a2rs, n_split=C)
        return kw

    def scratch_call(qkv, **kw):
        a = _cabi.LinearHArgs()
        for k, v in kw.items():
            setattr(a, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
        rc = scratch.bench_store_only(ctypes.byref(a), qkv, torch.cuda.current_stream().cuda_stream)
        assert rc == 0, "scratch launch failed"

    ku = L.round_up(INNER, 64)
    N_ff1, N_qkv = 2 * ku, 3 * C
    ff1 = operands(N_ff1, C, False)
    ff1["w_hi"], ff1["w_lo"], ff1["w_scale"] = L.split_f16_rs(L.pad_rows(
        L.pack_geglu(torch.rand(2 * INNER, C, device=dev, generator=g) * 0.1 - 0.05, INNER, ku), 256))
    U = torch.empty(2, M, N_ff1 // 2, dtype=torch.int16, device=dev)
    qkv = operands(N_qkv, C, True)
    P = torch.empty(2, M, N_qkv, dtype=torch.int16, device=dev)
    vinv = torch.empty(HEADS, M, device=dev)
    cos, sin = (t.to(dev).contiguous() for t in L.rope_tables(1024, C // HEADS))
    qs = torch.rand(C // HEADS, device=dev, generator=g) + 0.5
    ks = torch.rand(C // HEADS, device=dev, generator=g) + 0.5
    plain = operands(N_qkv, C, False)
    Cq = torch.empty(M, N_qkv, device=dev)

    kernels = [
        ("FF1 + GEGLU -> U planes", N_ff1, lambda: _cabi.linear_h(u_hi=U[0], u_lo=U[1], ldu=N_ff1 // 2,
                                                                  epilogue=_cabi.EPI_GEGLU, **ff1)),
        ("FF1 store-only", N_ff1, lambda: scratch_call(0, u_hi=U[0], u_lo=U[1], ldu=N_ff1 // 2, **ff1)),
        ("QKV -> planes", N_qkv, lambda: _cabi.linear_h(u_hi=P[0], u_lo=P[1], ldu=N_qkv, epilogue=_cabi.EPI_QKV_PLANES,
                                                        q_scale=qs, k_scale=ks, rope_cos=cos, rope_sin=sin,
                                                        qk_cols=2 * C, tokens=1024, q_plane_scale=2.0 ** 13,
                                                        k_plane_scale=2.0 ** 13, vinv=vinv, **qkv)),
        ("QKV store-only", N_qkv, lambda: scratch_call(1, u_hi=P[0], u_lo=P[1], ldu=N_qkv, qk_cols=2 * C, vinv=vinv,
                                                       **qkv)),
        ("qkv -> fp32 (plain)", N_qkv, lambda: _cabi.linear_h(c=Cq, ldc=N_qkv, epilogue=_cabi.EPI_NONE, **plain)),
    ]
    sms = props.multi_processor_count
    times = {name: [] for name, _, _ in kernels}
    for rnd in range(args.rounds):
        for name, N, fn in kernels:
            times[name].append(timeit(fn))
    for name, N, _ in kernels:
        tiles = (M + 127) // 128 * ((N + 127) // 128)
        per_cta = -(-tiles // sms)
        us = float(np.median(times[name]))
        print(f"{name:26s} M={M} N={N:5d} K=512  {us:8.1f} us  {per_cta} tiles a CTA  {us / per_cta:6.2f} us a tile"
              f"   rounds: {' '.join(f'{t:.1f}' for t in times[name])}", flush=True)
    for real, store in (("FF1 + GEGLU -> U planes", "FF1 store-only"), ("QKV -> planes", "QKV store-only")):
        N = N_ff1 if real.startswith("FF1") else N_qkv
        per_cta = -(-((M + 127) // 128 * ((N + 127) // 128)) // sms)
        gap = (np.median(times[real]) - np.median(times[store])) / per_cta
        print(f"epilogue gap {real}: {gap:.2f} us a tile over its store-only twin", flush=True)


if __name__ == "__main__":
    main()
