#!/usr/bin/env python
"""Kernel times of the row-wise kernels of csrc/rowwise.cu that the encode and decode run, each launched through its
entry point at a shape the package runs (cfg-3: 8 clips of 17 x 256^2, p = 8, pt = 4, C = 512, M = 40 960 tokens):
- omt_layernorm / omt_layernorm_h at M = 40 960 in the engine's three forms: fp32 in place; row-scaled planes of the
  normalised row; row-scaled planes of the normalised and the raw row.  C = 256, 512, 768 and 1024 reach the paired
  instantiations <2 | 4 | 6 | 8, true>; C = 128, 192, 384, 448 and 640 reach <1 | 2 | 3 | 4 | 8, false>;
- omt_layernorm in place with the patch embed's row map (its second LayerNorm), first frames and rest frames;
- omt_patchify_ln and omt_patchify_ln_u8 into row-scaled planes with LayerNorm, first frames (8 192 rows, K = 192) and
  rest frames (32 768 rows, K = 768), the uint8 gather also with VideoNorm's two tables picked per clip by sel; and the
  fp32 im2col form of patch_embed='cnn';
- omt_unpatchify and omt_unpatchify_u8 ((clamp(x + 0.5, 0, 1) * 255).byte()) of the cfg-3 decode, first and rest frames.

    python scripts/bench_rowwise.py [--rounds 15] [--reps 20]
    OMT_LIB=/path/to/libomnitok_b200.so python scripts/bench_rowwise.py      # another build of the same ABI

--reps launches are captured in one CUDA graph and the graph is replayed, so the time is the kernels' own.  Each
instance: one warm-up replay, then --rounds replays timed with CUDA events; the median, min and max over the rounds of
the time per launch, in microseconds.  The inputs are seeded and every output is hashed after the first launch (sha256,
first 16 hex digits of each output buffer), so two builds whose kernels give the same bits print the same hashes.
Prints ONE JSON line with the library, the card's name, power limit and max SM clock.
"""
import argparse
import hashlib
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from omnitokenizer_b200 import _cabi  # noqa: E402
from omnitokenizer_b200 import consumers as CS  # noqa: E402
from omnitokenizer_b200 import layout as L  # noqa: E402
from scripts.bench_ingest import card  # noqa: E402

DEV = torch.device("cuda:0")
EPS = 1e-5
B, T, S, CIN, P, PT = 8, 17, 256, 3, 8, 4           # cfg-3
N = (S // P) ** 2                                   # tokens per latent frame
TP = 1 + (T - 1) // PT                              # latent frames
M = B * TP * N                                      # 40 960 tokens
ROWS = {1: B * N, 0: B * (TP - 1) * N}             # patch rows of the first frames and of the rest
K = {1: CIN * P * P, 0: CIN * PT * P * P}          # 192, 768


def gen(seed):
    return torch.Generator().manual_seed(seed)


def f32(shape, seed, scale=1.0, offset=0.0):
    return (torch.randn(shape, generator=gen(seed)) * scale + offset).to(DEV)


def u8(shape, seed):
    return torch.randint(0, 256, shape, generator=gen(seed), dtype=torch.uint8).to(DEV)


def ln_params(C, seed):
    g = gen(seed)
    return (torch.rand(C, generator=g) + 0.5).to(DEV), ((torch.rand(C, generator=g) - 0.5) * 0.5).to(DEV)


def planes(rows, cols, rs=True):
    return (torch.empty(rows, cols, dtype=torch.int16, device=DEV), torch.empty(rows, cols, dtype=torch.int16, device=DEV),
            torch.empty(rows, device=DEV) if rs else None)


def layernorm(C, form):
    """form: 'fp32' (in place), 'y' (row-scaled planes of the normalised row), 'yx' (and of the raw row)."""
    x = f32((M, C), C, scale=4.0, offset=1.0)
    w, b = ln_params(C, C + 1)
    if form == "fp32":
        return [x], lambda: _cabi.call("omt_layernorm", x, C, x, C, w, b, M, C, EPS, 0, 0, 0)
    yp = planes(M, C)
    xp = planes(M, C) if form == "yx" else (None, None, None)
    outs = [t for t in yp + xp if t is not None]
    return outs, lambda: _cabi.call("omt_layernorm_h", x, C, None, 0, *yp, *xp, C, w, b, M, C, EPS, 0, 0, 0)


def layernorm_row_map(first):
    """The patch embed's second LayerNorm, in place on the rows of X its group's frames own."""
    C = 512
    x = f32((M, C), 7 + first, scale=4.0, offset=1.0)
    w, b = ln_params(C, 9)
    seg = (N, TP * N, 0) if first else ((TP - 1) * N, TP * N, N)
    return [x], lambda: _cabi.call("omt_layernorm", x, C, x, C, w, b, ROWS[first], C, EPS, *seg)


def gather(src, first, ln=True, with_sel=False):
    rows, k = ROWS[first], K[first]
    w, b = ln_params(k, 11 + first) if ln else (None, None)
    if ln:
        out = planes(rows, k)
        args = (None,) + out
    else:
        A = torch.empty(rows, k, device=DEV)
        out, args = (A,), (A, None, None, None)
    if src == "f32":
        video = f32((B, CIN, T, S, S), 13)
        return list(out), lambda: _cabi.call("omt_patchify_ln", video, *args, w, b, B, CIN, T, S, S, P, PT, first, EPS)
    frames = u8((B, T, S, S, CIN), 14)
    lut = L.u8_norm_table(CS.VIDEO_NORM if with_sel else CS.DIT_NORM, CIN).to(DEV)
    sel = (torch.arange(B, dtype=torch.int32) % 2).to(DEV) if with_sel else None
    return list(out), lambda: _cabi.call("omt_patchify_ln_u8", frames, lut, sel, *args, w, b, B, CIN, T, S, S, P, PT, first,
                                         EPS)


def unpatchify(first, to_u8):
    Pm = f32((ROWS[first], K[first]), 15 + first, scale=0.6)
    if to_u8:
        out = torch.zeros(B, T, S, S, CIN, dtype=torch.uint8, device=DEV)
        return [out], lambda: _cabi.call("omt_unpatchify_u8", Pm, out, B, CIN, T, S, S, P, PT, first, 1.0, 0.5, 0.0, 1.0,
                                         255.0)
    out = torch.zeros(B, CIN, T, S, S, device=DEV)
    return [out], lambda: _cabi.call("omt_unpatchify", Pm, out, B, CIN, T, S, S, P, PT, first)


CASES = {}
for _C, _inst in ((256, "<2, true>"), (512, "<4, true>"), (768, "<6, true>"), (1024, "<8, true>"), (128, "<1, false>"),
                  (192, "<2, false>"), (384, "<3, false>"), (448, "<4, false>"), (640, "<8, false>")):
    for _form in ("fp32", "y", "yx"):
        CASES[f"layernorm{_inst} C={_C} {_form}"] = (lambda C=_C, f=_form: layernorm(C, f))
for _first, _what in ((1, "first"), (0, "rest")):
    CASES[f"layernorm<4, true> patch row map {_what}"] = (lambda f=_first: layernorm_row_map(f))
    CASES[f"patchify_ln {_what} K={K[_first]} row-scaled"] = (lambda f=_first: gather("f32", f))
    CASES[f"patchify_ln_u8 {_what} K={K[_first]} row-scaled"] = (lambda f=_first: gather("u8", f))
    CASES[f"patchify_ln_u8 {_what} K={K[_first]} row-scaled sel"] = (lambda f=_first: gather("u8", f, with_sel=True))
    CASES[f"patchify_ln {_what} K={K[_first]} im2col"] = (lambda f=_first: gather("f32", f, ln=False))
    CASES[f"unpatchify {_what}"] = (lambda f=_first: unpatchify(f, False))
    CASES[f"unpatchify_u8 {_what}"] = (lambda f=_first: unpatchify(f, True))


def digest(outs):
    return [hashlib.sha256(t.cpu().numpy().tobytes()).hexdigest()[:16] for t in outs]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_rowwise.py measures on a GPU"
    torch.cuda.set_device(DEV)
    res = {}
    for name, make in CASES.items():
        outs, launch = make()
        launch()                                       # the call's checks and first launch, outside the capture
        torch.cuda.synchronize()
        hashes = digest(outs)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for _ in range(args.reps):
                launch()
        graph.replay()
        us = []
        for _ in range(args.rounds):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            graph.replay()
            b.record()
            b.synchronize()
            us.append(a.elapsed_time(b) * 1e3 / args.reps)
        res[name] = {"us": round(float(np.median(us)), 2), "min_max_us": [round(min(us), 2), round(max(us), 2)],
                     "sha256": hashes}
        del graph, outs, launch
        torch.cuda.empty_cache()
    print(json.dumps({"metric": "rowwise_kernel_us", "lib": _cabi.lib_path(), "rounds": args.rounds, "reps": args.reps,
                      "card": card(), "instances": res}))


if __name__ == "__main__":
    main()
