#!/usr/bin/env python
"""The FVD leg of vqgan_eval.py's video loop with --infer_downsample 2 for one cfg-3 eval batch (8 clips x 17 x 256^2),
seeded tokenizer and seeded I3D weights (oracle/i3d_oracle.py weights with the BatchNorm statistics of
tests/golden/fvd_i3d.pt).

    python scripts/bench_eval_downsample.py [--rounds 5] [--d 2]

Arms, in alternating rounds in one process, each step ending in a synchronise:
- (a) consumers.eval_step_fvd without the flag (the full-resolution scores);
- (b) consumers.eval_step_fvd with infer_downsample=d: forward_u8's fp32 reconstruction and the real clip through
  omt_eval_downsample, then both I3D calls on the device;
- (c) the script's host path (vqgan_eval.py:121-148): forward_u8's fp32 reconstruction to the host, the clamp, torch's
  CPU F.interpolate of both sides (default threads), * 255 .byte(), and fvd.get_fvd_logits from the numpy arrays.
Reports ms per batch of each arm, whether (b) and (c) give the same logits bit for bit, and the downsample kernel's
device time (CUDA events, both sides).  Prints ONE JSON line with the card's name, power limit and max SM clock.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import omnitokenizer_b200 as ob  # noqa: E402
from omnitokenizer_b200 import consumers as C  # noqa: E402
from omnitokenizer_b200 import downsample, fvd  # noqa: E402
from omnitokenizer_b200 import layout as L  # noqa: E402
from oracle import i3d_oracle as io  # noqa: E402
from oracle import omni_oracle as oo  # noqa: E402
from oracle import weights as W  # noqa: E402
from scripts.bench_ingest import card  # noqa: E402

B, T, S = 8, 17, 256


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--d", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_eval_downsample.py measures on a GPU"
    dev = torch.device("cuda:0")
    d = args.d

    margs = ob.canonical_args()
    m = ob.OmniTokenizer_VQGAN(margs)
    m.load_state_dict(W.make_state_dict(oo.Config.from_args(margs), 0), strict=False)
    m.codebook._need_init = False
    m = m.to(dev).eval()
    golden = torch.load(os.path.join(ROOT, "tests", "golden", "fvd_i3d.pt"))
    sd = io.make_state_dict(golden["w_seed"])
    sd.update(golden["bn"])
    i3d = fvd.I3D(sd, dev)

    u8 = torch.randint(0, 256, (B, T, S, S, 3), generator=torch.Generator().manual_seed(1), dtype=torch.uint8)
    frames = u8.to(dev)
    video = L.u8_normalize(u8, C.VIDEO_NORM)              # the loader's normalised clip, (B, 3, T, H, W) fp32, host

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, out

    def arm_a():
        return C.eval_step_fvd(m, frames, i3d)[:2]

    def arm_b():
        return C.eval_step_fvd(m, frames, i3d, infer_downsample=d)[:2]

    def arm_c():
        with torch.no_grad():
            x_recons, _ = m.forward_u8(frames, C.VIDEO_NORM, None)
            real_videos = video + 0.5
            fake_videos = torch.clamp(x_recons.cpu() + 0.5, 0, 1)
            sides = []
            for v in (real_videos, fake_videos):
                v = v.permute(0, 2, 1, 3, 4).flatten(0, 1)
                v = F.interpolate(v, scale_factor=1 / d, mode="bilinear", align_corners=False)
                v = v.unflatten(0, (B, T)).permute(0, 2, 1, 3, 4)
                sides.append(fvd.get_fvd_logits((v * 255).movedim(1, -1).byte().numpy(), i3d, dev).clone())
        return tuple(sides)

    arms = {"a_full_res": arm_a, "b_downsample_gpu": arm_b, "c_downsample_host": arm_c}
    for _ in range(2):                                     # warm-up: graphs captured, descriptors uploaded
        for fn in arms.values():
            fn()
    times = {k: [] for k in arms}
    outs = {}
    for _ in range(args.rounds):
        for k, fn in arms.items():
            ms, outs[k] = timed(fn)
            times[k].append(ms)
    med = {k: float(np.median(v)) for k, v in times.items()}

    # the downsample kernel alone, both sides, CUDA events over 20 repetitions
    x_recons, _ = m.forward_u8(frames, C.VIDEO_NORM, None)
    downsample.clips_u8(frames, d, real_norm=C.VIDEO_NORM)
    a_ev, b_ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a_ev.record()
    for _ in range(20):
        downsample.clips_u8(frames, d, real_norm=C.VIDEO_NORM)
        downsample.clips_u8(x_recons, d)
    b_ev.record()
    torch.cuda.synchronize()
    kernel_ms = a_ev.elapsed_time(b_ev) / 20
    bytes_moved = frames.numel() + x_recons.numel() * 4 + 2 * B * T * (S // d) ** 2 * 3

    same = all(torch.equal(x, y) for x, y in zip(outs["b_downsample_gpu"], outs["c_downsample_host"]))
    out = {
        "metric": "eval_downsample_ms_per_batch", "workload": f"cfg3 eval batch: {B} clips {T}x{S}x{S}, d={d}",
        "rounds": args.rounds, "median_ms": {k: round(v, 2) for k, v in med.items()},
        "spread_ms": {k: [round(min(v), 2), round(max(v), 2)] for k, v in times.items()},
        "host_over_gpu": round(med["c_downsample_host"] / med["b_downsample_gpu"], 2),
        "downsample_over_full_res": round(med["b_downsample_gpu"] / med["a_full_res"], 3),
        "b_equals_c_bitwise": same, "kernel_ms_both_sides": round(kernel_ms, 4),
        "kernel_min_bytes_gb_per_s": round(bytes_moved / (kernel_ms * 1e-3) / 1e9, 1),
        "torch_threads": torch.get_num_threads(), "card": card(),
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
