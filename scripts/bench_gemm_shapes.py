"""CUDA-event timing of the model's GEMM shapes (L2 flushed between launches, median of 7 launches):
   python scripts/bench_gemm_shapes.py [M ...]      -> one line per (form, shape): us, algorithmic TFLOP/s, fraction of tf32 peak
   python scripts/bench_gemm_shapes.py --ksweep     -> FF1 + GEGLU and QKV -> planes (row-scaled) at M = 40 960 over
                                                       K = 512, 1024, 2048, fitted to t(K) = a + b K
   ... --lib A.so --lib B.so [--rounds R]           -> same-process A/B of several builds of the library: every shape is
                                                       timed on each build in turn, R rounds alternating, and the outputs
                                                       of every build are compared bit for bit with the first one's

Forms: "rs" = the row-scaled single-accumulator f16x3 GEMM (LayerNorm / patch-gather fed), "2^11" = the two-accumulator
f16x3 GEMM (2^11-scaled lo planes), "3xtf32" = the fp32-operand GEMM, "rs-h1" / "2^11-h1" = the single-product f16x1
GEMM (omt_linear_h1) on the hi planes of the same operands.  These are the gemm_wgmma_kernel forms the engine launches.  In the K sweep the intercept a is the per-launch cost that does not grow with K: with a persistent grid
it is mostly the per-tile work that the mainloop does not hide (the epilogue) plus the pipeline fill."""
import argparse
import ctypes
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from omnitokenizer_b200 import _cabi, layout as L  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("M", type=int, nargs="*", default=[40960, 5120])
ap.add_argument("--ksweep", action="store_true")
ap.add_argument("--lib", action="append", default=[], help="library build to time (repeat for an A/B; default: in-tree)")
ap.add_argument("--rounds", type=int, default=1, help="alternating rounds over the builds")
args = ap.parse_args()

dev = torch.device("cuda:0")
# tf32 dense = half the dense bf16 rate; without a measured peak, the H100 SXM data sheet's 989 TFLOP/s bf16 (as bench.py)
pk = (json.load(open("MEASURED_PEAKS.json"))["bf16_tflops"] if os.path.exists("MEASURED_PEAKS.json") else 989.0) / 2
flush = torch.zeros(64 * 1024 * 1024, device=dev)

def load_lib(path):
    lib = ctypes.CDLL(os.path.abspath(path))
    for name, (res, argtypes) in _cabi.SIGNATURES.items():
        fn = getattr(lib, name, None)     # an older build lacks the newer entry points; its forms are timed without them
        if fn is not None:
            fn.restype, fn.argtypes = res, argtypes
    assert lib.omt_abi_version() == _cabi.ABI_VERSION, f"{path}: ABI version mismatch"
    return lib


LIBS = [(os.path.basename(os.path.dirname(os.path.abspath(p))) + "/" + os.path.basename(p), load_lib(p))
        for p in (args.lib or [_cabi.lib_path()])]
C, INNER, HEADS = 512, 1365, 8


def timeit(fn, reps=7):
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for i in range(reps + 2):
        flush.add_(1.0)
        if i >= 2: evs[i - 2][0].record()
        fn()
        if i >= 2: evs[i - 2][1].record()
    torch.cuda.synchronize()
    return sorted(a.elapsed_time(b) for a, b in evs)[reps // 2] * 1e3


def make(kind, form, M, K, g):
    """(launch, N, outputs) of one GEMM of the model: kind in qkv (plain C), qkv-planes, out+res, ff1+geglu, ff2+res."""
    mult = 32 if form == "3xtf32" else 64
    if kind == "ff1+geglu":
        ku = L.round_up(INNER, mult); Np = 2 * ku; Kp = K
        W = L.pack_geglu(torch.rand(2 * INNER, K, device=dev, generator=g) * 0.1 - 0.05, INNER, ku)
    else:
        Np = {"qkv": 3 * C, "qkv-planes": 3 * C, "out+res": C, "ff2+res": C}[kind]; Kp = L.round_up(K, mult)
        W = L.pad_cols(torch.rand(Np, K, device=dev, generator=g) * 0.1 - 0.05, Kp)
    A = torch.rand(M, Kp, device=dev, generator=g) - 0.5
    R = torch.rand(M, C, device=dev, generator=g)
    if form == "3xtf32":
        Wp = L.pad_rows(W, 128); hi = L.tf32_round(Wp); lo = (Wp - hi).contiguous()
        if kind == "ff1+geglu":
            U = torch.empty(M, Np // 2, device=dev)
            return lambda: _cabi.call("omt_linear", A, Kp, 0, 0, 0, hi, lo, U, Np // 2, 0, 0, 0, M, Np, Kp, None, None, 0, _cabi.EPI_GEGLU, _cabi.MATH_3XTF32), Np, [U]
        if kind in ("qkv", "qkv-planes"):
            Cq = torch.empty(M, Np, device=dev)
            return lambda: _cabi.call("omt_linear", A, Kp, 0, 0, 0, hi, lo, Cq, Np, 0, 0, 0, M, Np, Kp, None, None, 0, _cabi.EPI_NONE, _cabi.MATH_3XTF32), Np, [Cq]
        return lambda: _cabi.call("omt_linear", A, Kp, 0, 0, 0, hi, lo, R, C, 0, 0, 0, M, Np, Kp, None, R, C, _cabi.EPI_NONE, _cabi.MATH_3XTF32), Np, [R]
    h1 = form.endswith("-h1")
    if form.startswith("rs"):
        ah, al, ars = L.split_rows_rs(A); wh, wl, wsc = L.split_f16_rs(L.pad_rows(W, 256)); kw = dict(a_rs=ars, w_scale=wsc)
    else:
        ah, al = L.split_f16(A); wh, wl = L.split_f16(L.pad_rows(W, 256)); kw = {}
    kw.update(a_hi=ah, a_lo=al, lda=Kp, w_hi=wh, w_lo=wl, M=M, N=Np, K=Kp)

    def linear_h(**k):     # omt_linear_h, or omt_linear_h1 with the lo planes left out
        if h1:
            return _cabi.linear_h("omt_linear_h1", **{f: v for f, v in k.items() if f not in ("a_lo", "a2_lo", "w_lo", "u_lo")})
        return _cabi.linear_h(**k)
    if kind == "ff1+geglu":
        U = torch.empty(2, M, Np // 2, dtype=torch.int16, device=dev)
        return lambda: linear_h(u_hi=U[0], u_lo=U[1], ldu=Np // 2, epilogue=_cabi.EPI_GEGLU, **kw), Np, [U]
    if kind == "qkv-planes":
        # the spatial-attention layer's launch: q from the normalised rows, k / v from the raw rows (dual A), rope +
        # l2norm + scale on q / k, q | k | v written as operand planes, N = 1024 tokens per frame
        a2h, a2l, a2rs = (L.split_rows_rs(A.flip(1)) if form.startswith("rs") else L.split_f16(A.flip(1)) + (None,))
        cos, sin = (t.to(dev).contiguous() for t in L.rope_tables(1024, C // HEADS))
        qs = torch.rand(C // HEADS, device=dev, generator=g) + 0.5; ks = torch.rand(C // HEADS, device=dev, generator=g) + 0.5
        U = torch.empty(2, M, Np, dtype=torch.int16, device=dev); vinv = torch.empty(HEADS, M, device=dev)
        return lambda: linear_h(a2_hi=a2h, a2_lo=a2l, a2_rs=a2rs, n_split=C, u_hi=U[0], u_lo=U[1], ldu=Np,
                                      epilogue=_cabi.EPI_QKV_PLANES, q_scale=qs, k_scale=ks, rope_cos=cos, rope_sin=sin,
                                      qk_cols=2 * C, tokens=1024, q_plane_scale=2.0 ** 13, k_plane_scale=2.0 ** 13, vinv=vinv,
                                      **kw), Np, [U, vinv]
    if kind == "qkv":
        Cq = torch.empty(M, Np, device=dev)
        return lambda: linear_h(c=Cq, ldc=Np, epilogue=_cabi.EPI_NONE, **kw), Np, [Cq]
    return lambda: linear_h(c=R, ldc=C, residual=R, ldr=C, epilogue=_cabi.EPI_NONE, **kw), Np, [R]


def run(kind, form, M, N, K):
    """Times the shape on every build (args.rounds alternating rounds) and returns the first build's median."""
    fn, Np, outs = make(kind, form, M, K, torch.Generator(device=dev).manual_seed(1))
    R0 = outs[0].clone() if kind in ("out+res", "ff2+res") else None
    ref = None
    times = {name: [] for name, _ in LIBS}
    for rnd in range(args.rounds):
        for name, lib in LIBS:
            _cabi._lib = lib
            us = timeit(fn)
            if R0 is not None:
                outs[0].copy_(R0)         # the residual forms accumulate into R: one more launch from the initial R
            fn()
            times[name].append(us)
            got = [o.clone() for o in outs]
            if ref is None:
                ref = got
            same = all(torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a,
                                   b.view(torch.int32) if b.dtype == torch.float32 else b) for a, b in zip(got, ref))
            tf = 2.0 * M * N * K / us / 1e6
            tag = f"  {name}  round {rnd}  {'same bits' if same else 'OUTPUT DIFFERS from the first build'}" if len(LIBS) > 1 else ""
            print(f"{form:6s} M={M:6d} {kind:10s} N={Np:5d} K={K:5d} {us:8.1f} us  {tf:7.1f} TFLOP/s  {tf / pk:.3f} of tf32 peak{tag}",
                  flush=True)
    if len(LIBS) > 1:
        meds = {name: float(np.median(t)) for name, t in times.items()}
        base = meds[LIBS[0][0]]
        print("   median: " + "  ".join(f"{name} {us:.1f} us ({base / us:.3f}x the first build's speed)"
                                      for name, us in meds.items()), flush=True)
    return float(np.median(times[LIBS[0][0]]))


print(f"device: {torch.cuda.get_device_name(dev)}", flush=True)
if args.ksweep:
    Ks = [512, 1024, 2048]
    for kind, N in (("ff1+geglu", 2 * INNER), ("qkv-planes", 3 * C)):
        t = [run(kind, "rs", 40960, N, K) for K in Ks]
        b, a = np.polyfit(Ks, t, 1)
        print(f"fit {kind}: t(K) = {a:.1f} us + {b * 1e3:.2f} us per 1000 K;  a / t(512) = {a / t[0]:.1%}", flush=True)
else:
    SHAPES = [("qkv", 3 * C, C), ("qkv-planes", 3 * C, C), ("out+res", C, C), ("ff1+geglu", 2 * INNER, C), ("ff2+res", C, INNER)]
    for M in args.M:
        for kind, N, K in SHAPES:
            for form in ("rs", "rs-h1", "2^11", "2^11-h1", "3xtf32"):
                if kind == "qkv-planes" and form == "3xtf32":
                    continue
                run(kind, form, M, N, K)
