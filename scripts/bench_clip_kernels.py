#!/usr/bin/env python
"""Kernel times of the bilinear clip kernel (csrc/resample.cu, bilinear_clips_kernel) at each of its ten
instantiations, each launched through its entry point at a shape the package runs:
- omt_resample_clips: Latte's ucf101 config, 5 clips x 17 frames of 240 x 320 -> 256^2, alternate clips flipped;
- omt_fvd_preprocess: one cfg-3 eval batch, 8 x 17 x 256^2 -> 224^2, with one byte table, and with VideoNorm's two
  tables picked per clip by sel;
- omt_fid_preprocess: pytorch-fid's batch of 50 images, 256^2 -> 299^2;
- omt_fvd_suite_preprocess: 8 clips of 17 x 128^2 -> 224^2 (the suite's preprocess_single geometry), uint8, fp32 and
  videogpt's truncated fp32;
- omt_is_preprocess: one chunk of 64 frames at 299^2, resized from 256^2 and at their own size, uint8 and fp32;
- omt_eval_downsample: one cfg-3 eval batch with --infer_downsample 2, 8 x 17 x 256^2 -> 128^2, both sides.

    python scripts/bench_clip_kernels.py [--rounds 15] [--reps 20]
    OMT_LIB=/path/to/libomnitok_b200.so python scripts/bench_clip_kernels.py      # another build of the same ABI

The entry points check their descriptors on the host at every call, so --reps launches are captured in one CUDA graph
and the graph is replayed: the time is the kernels' own.  Each instance: one warm-up replay, then --rounds replays
timed with CUDA events; the median, min and max over the rounds of the time per launch, in microseconds.  The inputs
are seeded, so the sha256 of each output (first 16 hex digits) is equal on two builds whose kernels give the same
bits.  Prints ONE JSON line with the library, the card's name, power limit and max SM clock.
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

from omnitokenizer_b200 import _cabi, downsample, fid, fvd, iscore  # noqa: E402
from omnitokenizer_b200 import consumers as C  # noqa: E402
from omnitokenizer_b200 import layout as L  # noqa: E402
from omnitokenizer_b200.metricnet import (FORM_F32, FORM_F32_TRUNC, FORM_U8, axis_tables, byte_lut,  # noqa: E402
                                          clip_descs, real_byte_table)
from scripts.bench_ingest import card  # noqa: E402

DEV = torch.device("cuda:0")


def u8(shape, seed):
    return torch.randint(0, 256, shape, generator=torch.Generator().manual_seed(seed), dtype=torch.uint8).to(DEV)


def f32(shape, seed):
    return torch.rand(shape, generator=torch.Generator().manual_seed(seed)).to(DEV)


def tables(desc_host, tab_host):
    return desc_host.to(DEV), desc_host, tab_host.to(DEV), tab_host, tab_host.numel()


def latte():
    B, F, H, W, S = 5, 17, 240, 320, 256
    g = L.clip_geometry(H, W, L.ucf_clip_resize(S))
    tab_host = torch.from_numpy(np.concatenate([L.clip_axis_table(g.wh, g.rh, g.scale_h).reshape(-1),
                                                L.clip_axis_table(g.ww, g.rw, g.scale_w).reshape(-1)]))
    desc_host = clip_descs(B, F * H * W * 3, H, W, g.rh, g.rw, g.cy, g.cx)
    desc_host[:, 4:8] = torch.tensor([g.y0, g.x0, g.wh, g.ww], dtype=torch.int32)
    desc_host[:, 12] = torch.arange(B) % 2
    desc_host[:, 15] = L.clip_interp_form(g, L.ucf_clip_resize(S).in_workers)
    src, norm, t = u8((B, F, H, W, 3), 1), L.clip_norm_table(C.LATTE_NORM).to(DEV), tables(desc_host, tab_host)
    out = torch.empty(B, 3, F, S, S, device=DEV)
    return out, lambda: _cabi.call("omt_resample_clips", src, src.numel(), *t, norm, B, F, S, S, out)


def fvd_case(with_sel):
    B, T, S = 8, 17, 256
    (oh, ow), src = fvd.TARGET_RESOLUTION, u8((B, T, S, S, 3), 2)
    lut = (real_byte_table(C.VIDEO_NORM).float() if with_sel else byte_lut()[0] * 255).to(DEV)
    sel = (torch.arange(B, dtype=torch.int32) % 2).to(DEV) if with_sel else None
    t = tables(clip_descs(B, T * S * S * 3, S, S, oh, ow), axis_tables(S, S, oh, ow))
    out = torch.empty(B, T, oh, ow, 4, device=DEV)
    return out, lambda: _cabi.call("omt_fvd_preprocess", src, src.numel(), *t, lut, sel, B, T, oh, ow, out)


def fid_case():
    B, S = 50, 256
    (oh, ow), src, lut = fid.TARGET_RESOLUTION, u8((B, S, S, 3), 3), byte_lut()[0].to(DEV)
    t = tables(clip_descs(B, S * S * 3, S, S, oh, ow), axis_tables(S, S, oh, ow))
    out = torch.empty(B, oh, ow, 4, device=DEV)
    return out, lambda: _cabi.call("omt_fid_preprocess", src, src.numel(), *t, lut, None, B, oh, ow, out)


def suite_case(form):
    B, T, S = 8, 17, 128
    c = fvd.SuiteClips(u8((B, T, S, S, 3), 4) if form == FORM_U8 else f32((B, T, 3, S, S), 4), form)
    (oh, ow) = fvd.TARGET_RESOLUTION
    out = torch.empty(B, T, oh, ow, 4, device=DEV)
    return out, lambda: _cabi.call("omt_fvd_suite_preprocess", c.src, c.src.numel(), form, c.C, c.desc, c.desc_host,
                                   c.tab, c.tab_host, c.tab_host.numel(), B, T, oh, ow, out)


def is_case(form, resize):
    N, S = 64, 256 if resize else 299
    src = u8((N, S, S, 3), 5) if form == FORM_U8 else f32((N, 3, S, S), 5)
    oh, ow = iscore.TARGET_RESOLUTION
    t = tables(clip_descs(N, 3 * S * S, S, S, oh, ow), axis_tables(S, S, *((oh, ow) if resize else (None, None))))
    out = torch.empty(N, oh, ow, 4, device=DEV)
    return out, lambda: _cabi.call("omt_is_preprocess", src, src.numel(), form, *t, N, 1, oh, ow, out)


def eval_case(form):
    B, T, S, d = 8, 17, 256, 2
    oh, ow = downsample.out_size(S, S, d)
    desc_host, tab_host, desc, tab = downsample._interp_setup(B, T, S, S, d, False, DEV)
    t = (desc, desc_host, tab, tab_host, tab_host.numel())
    if form == downsample.FORM_U8:
        src, lut = u8((B, T, S, S, 3), 6), downsample.real_value_table(C.VIDEO_NORM).to(DEV)
        sel = (torch.arange(B, dtype=torch.int32) % 2).to(DEV)
    else:
        src, lut, sel = f32((B, 3, T, S, S), 6) * 2 - 1.5, None, None
    out = torch.empty(B, T, oh, ow, 3, dtype=torch.uint8, device=DEV)
    return out, lambda: _cabi.call("omt_eval_downsample", src, src.numel(), form, *t, lut, sel, B, T, oh, ow, out)


CASES = {
    "resample_clips (ByteTable, NormalizePlanes) ucf 5x17 240x320->256": latte,
    "fvd_preprocess (ByteTable, Float4 2y/255-1) 8x17 256->224": lambda: fvd_case(False),
    "fvd_preprocess sel": lambda: fvd_case(True),
    "fid_preprocess (ByteTable, Float4 2y-1) 50 256->299": fid_case,
    "fvd_suite u8 (SuiteFrames<U8>, Float4 (y-0.5)2) 8x17 128->224": lambda: suite_case(FORM_U8),
    "fvd_suite f32 (SuiteFrames<F32>)": lambda: suite_case(FORM_F32),
    "fvd_suite f32 trunc (SuiteFrames<F32_TRUNC>)": lambda: suite_case(FORM_F32_TRUNC),
    "is u8 (SuiteFrames<U8>, Float4 y) 64 256->299": lambda: is_case(FORM_U8, True),
    "is u8 64 299 no resize": lambda: is_case(FORM_U8, False),
    "is f32 (SuiteFrames<F32>, Float4 y) 64 256->299": lambda: is_case(FORM_F32, True),
    "is f32 64 299 no resize": lambda: is_case(FORM_F32, False),
    "eval_downsample u8 (ByteTable, BytePixels) 8x17 256->128": lambda: eval_case(downsample.FORM_U8),
    "eval_downsample f32 (ClampedPlanes, BytePixels)": lambda: eval_case(downsample.FORM_F32),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_clip_kernels.py measures on a GPU"
    torch.cuda.set_device(DEV)
    res = {}
    for name, make in CASES.items():
        out, launch = make()
        launch()                                       # the call's checks and first launch, outside the capture
        torch.cuda.synchronize()
        digest = hashlib.sha256(out.cpu().numpy().tobytes()).hexdigest()[:16]
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
        same = hashlib.sha256(out.cpu().numpy().tobytes()).hexdigest()[:16] == digest
        res[name] = {"us": round(float(np.median(us)), 2), "min_max_us": [round(min(us), 2), round(max(us), 2)],
                     "sha256": digest, "replay_same_bytes": same}
        del graph, out, launch
        torch.cuda.empty_cache()
    print(json.dumps({"metric": "clip_kernel_us", "lib": _cabi.lib_path(), "rounds": args.rounds, "reps": args.reps,
                      "card": card(), "instances": res}))


if __name__ == "__main__":
    main()
