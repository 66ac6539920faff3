"""CUDA-event timing of the model's GEMM shapes (L2 flushed between launches) for the tensor-core math modes:
   python scripts/bench_gemm_shapes.py [M ...]      -> one line per (math, shape): us, algorithmic TFLOP/s, fraction of tf32 peak"""
import json, os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from omnitokenizer_b200 import _cabi, layout as L

dev = torch.device("cuda:0")
Ms = [int(a) for a in sys.argv[1:]] or [40960, 5120]
# tf32 dense = half the dense bf16 rate; without a measured peak, the H100 SXM data sheet's 989 TFLOP/s bf16 (as bench.py)
pk = (json.load(open("MEASURED_PEAKS.json"))["bf16_tflops"] if os.path.exists("MEASURED_PEAKS.json") else 989.0) / 2
flush = torch.zeros(64 * 1024 * 1024, device=dev)
_cabi.load()


def timeit(fn, reps=7):
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for i in range(reps + 2):
        flush.add_(1.0)
        if i >= 2: evs[i - 2][0].record()
        fn()
        if i >= 2: evs[i - 2][1].record()
    torch.cuda.synchronize()
    return sorted(a.elapsed_time(b) for a, b in evs)[reps // 2] * 1e3


SHAPES = [("qkv", 1536, 512, "qkv"), ("out+res", 512, 512, "res"), ("ff1+geglu", 2730, 512, "geglu"), ("ff2+res", 512, 1365, "res")]
for scheme in [int(v) for v in os.environ.get("F16_BN", "256,128,1").split(",")]:       # 1 = row-scaled single-accumulator form
  _cabi.set_option("f16_bn", scheme if scheme > 1 else 0)
  for M in Ms:
    for name, N, K, kind in SHAPES:
        g = torch.Generator(device=dev).manual_seed(1)
        for math in (("3xtf32", "f16x3") if scheme == 256 else ("f16x3",)):
            mult = 64 if math == "f16x3" else 32
            if kind == "geglu":
                inner = 1365; ku = L.round_up(inner, mult); Np = 2 * ku; Kp = K
                W = L.pack_geglu(torch.rand(2 * inner, K, device=dev, generator=g) * 0.1 - 0.05, inner, ku)
            else:
                Kp = L.round_up(K, mult); Np = N
                W = L.pad_cols(torch.rand(N, K, device=dev, generator=g) * 0.1 - 0.05, Kp)
            A = torch.rand(M, Kp, device=dev, generator=g) - 0.5
            R = torch.rand(M, 512, device=dev, generator=g)
            flops = 2.0 * M * N * K
            if math == "3xtf32":
                Wp = L.pad_rows(W, 128); hi = L.tf32_round(Wp); lo = (Wp - hi).contiguous()
                if kind == "geglu":
                    U = torch.empty(M, Np // 2, device=dev)
                    fn = lambda: _cabi.call("omt_linear", A, Kp, 0, 0, 0, hi, lo, U, Np // 2, 0, 0, 0, M, Np, Kp, None, None, 0, _cabi.EPI_GEGLU, _cabi.MATH_3XTF32)
                elif kind == "qkv":
                    C = torch.empty(M, Np, device=dev)
                    fn = lambda: _cabi.call("omt_linear", A, Kp, 0, 0, 0, hi, lo, C, Np, 0, 0, 0, M, Np, Kp, None, None, 0, _cabi.EPI_NONE, _cabi.MATH_3XTF32)
                else:
                    fn = lambda: _cabi.call("omt_linear", A, Kp, 0, 0, 0, hi, lo, R, 512, 0, 0, 0, M, Np, Kp, None, R, 512, _cabi.EPI_NONE, _cabi.MATH_3XTF32)
            else:
                rsk = {}
                if scheme == 1:
                    ah, al, ars = L.split_rows_rs(A); wh, wl, wsc = L.split_f16_rs(L.pad_rows(W, 256)); rsk = dict(a_rs=ars, w_scale=wsc)
                else:
                    ah, al = L.split_f16(A); wh, wl = L.split_f16(L.pad_rows(W, 256))
                if kind == "geglu":
                    U = torch.empty(2, M, Np // 2, dtype=torch.int16, device=dev)
                    fn = lambda: _cabi.linear_h(a_hi=ah, a_lo=al, lda=Kp, w_hi=wh, w_lo=wl, u_hi=U[0], u_lo=U[1], ldu=Np // 2, M=M, N=Np, K=Kp, epilogue=_cabi.EPI_GEGLU, **rsk)
                elif kind == "qkv":
                    C = torch.empty(M, Np, device=dev)
                    fn = lambda: _cabi.linear_h(a_hi=ah, a_lo=al, lda=Kp, w_hi=wh, w_lo=wl, c=C, ldc=Np, M=M, N=Np, K=Kp, epilogue=_cabi.EPI_NONE, **rsk)
                else:
                    fn = lambda: _cabi.linear_h(a_hi=ah, a_lo=al, lda=Kp, w_hi=wh, w_lo=wl, c=R, ldc=512, M=M, N=Np, K=Kp, residual=R, ldr=512, epilogue=_cabi.EPI_NONE, **rsk)
            try:
                us = timeit(fn)
                tf = flops / us / 1e6
                print(f"bn{scheme} M={M:6d} {name:10s} {math:7s} {us:8.1f} us  {tf:7.1f} TFLOP/s  {tf / pk:.3f} of tf32 peak", flush=True)
            except Exception as e:
                print(f"bn{scheme} M={M} {name} {math} FAILED: {e}", flush=True)
                raise
