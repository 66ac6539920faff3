#!/usr/bin/env python
"""Mixed batches: one packed pass (encode_batch + decode_batch) against the passes a caller makes without it.

    python scripts/bench_mixed.py [--workloads joint,lengths] [--reps 5] [--math f16x3]

Workloads at 256 x 256 (bench.py's model, f16x3 by default):
- joint:   8 images + 4 clips of 17 frames (the LM stage's --loader_type joint data);
- lengths: 2 clips each of 9, 17, 33 and 65 frames (T' = 3, 5, 9, 17).
Each is encoded and decoded three ways: (a) one encode + decode per sample, (b) one per distinct shape (the samples of a
shape stacked into one batch), (c) encode_batch + decode_batch over the whole list.  Every way runs twice untimed (the
first call of a shape runs eagerly, the second captures its CUDA graph; each way has its own model, so its own resident
workspaces and graphs), then --reps timed rounds alternate (a), (b), (c), rotating which way starts a round (a card
that lowers its clocks under sustained load would otherwise favour whichever way runs first); each time is the host clock around a round that ends in a device synchronise.  frames/s counts an image as one frame.
The codes and reconstructions of the three ways are compared bit for bit.  Prints ONE JSON line per workload with the
card's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clk = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:          # the measurement still stands; the card is then named by torch only
        return {"name": torch.cuda.get_device_name(), "power_limit": f"unknown ({e.__class__.__name__})"}


def workload(name, dev):
    g = torch.Generator().manual_seed(7)
    if name == "joint":
        shapes = [(3, 256, 256)] * 8 + [(3, 17, 256, 256)] * 4
    else:
        shapes = [(3, t, 256, 256) for t in (9, 17, 33, 65) for _ in range(2)]
    # interleave images and clips as a loader would hand them over
    order = sorted(range(len(shapes)), key=lambda i: (i % 3, i))
    return [(torch.rand(shapes[i], generator=g) - 0.5).to(dev) for i in order]


def per_sample(m, xs):
    codes = [m.encode(x[None], x.ndim == 3)[0] for x in xs]
    recs = [m.decode(c[None], x.ndim == 3)[0] for x, c in zip(xs, codes)]
    return codes, recs


def per_shape(m, xs):
    buckets = {}
    for i, x in enumerate(xs):
        buckets.setdefault(tuple(x.shape), []).append(i)
    codes, recs = [None] * len(xs), [None] * len(xs)
    for shape, idx in buckets.items():
        img = len(shape) == 3
        c = m.encode(torch.stack([xs[i] for i in idx]), img)
        r = m.decode(c, img)
        for k, i in enumerate(idx):
            codes[i], recs[i] = c[k], r[k]
    return codes, recs


def packed(m, xs):
    codes = m.encode_batch(xs)
    return codes, m.decode_batch(codes)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="joint,lengths")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--math", default="f16x3")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mixed.py measures on a CUDA device; none is visible")
    os.environ["OMT_MATH"] = args.math
    import bench
    dev = torch.device("cuda:0")
    info = card()
    ways = {"a_per_sample": per_sample, "b_per_shape": per_shape, "c_packed": packed}
    # one model (same seeded weights) per way: each keeps its own resident workspaces and graphs, as a caller that only
    # ever uses that way would see them
    models = {name: bench.make_model(dev) for name in ways}
    for wl in args.workloads.split(","):
        xs = workload(wl, dev)
        frames = sum(1 if x.ndim == 3 else x.shape[1] for x in xs)
        out = {}
        for name, fn in ways.items():
            for _ in range(2):
                out[name] = fn(models[name], xs)
        torch.cuda.synchronize()
        ref_codes, ref_recs = out["a_per_sample"]
        equal = {}
        for name, (codes, recs) in out.items():
            c = [cc.reshape(r.shape) for cc, r in zip(codes, ref_codes)]     # packed image codes come without the frame axis
            equal[name] = all(torch.equal(a, b) for a, b in zip(c, ref_codes)) and all(torch.equal(a, b) for a, b in zip(recs, ref_recs))
        times = {name: [] for name in ways}
        names = list(ways)
        for rep in range(args.reps):
            for name in names[rep % 3:] + names[:rep % 3]:      # rotate which way runs first in a round
                fn = ways[name]
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn(models[name], xs)
                torch.cuda.synchronize()
                times[name].append(time.perf_counter() - t0)
        res = {"workload": wl, "math": args.math, "samples": len(xs), "frames": frames,
               "shapes": sorted({tuple(x.shape) for x in xs}), "outputs_equal": equal, "card": info}
        for name, ts in times.items():
            ts = sorted(ts)
            res[name] = {"frames_per_s": round(frames / ts[len(ts) // 2], 1), "ms_median": round(1e3 * ts[len(ts) // 2], 2),
                         "ms_min": round(1e3 * ts[0], 2), "ms_max": round(1e3 * ts[-1], 2)}
        res["speedup_c_over_a"] = round(res["c_packed"]["frames_per_s"] / res["a_per_sample"]["frames_per_s"], 3)
        res["speedup_c_over_b"] = round(res["c_packed"]["frames_per_s"] / res["b_per_shape"]["frames_per_s"], 3)
        print(json.dumps(res), flush=True)
        if not all(equal.values()):
            raise SystemExit(f"{wl}: the three ways disagree: {equal}")


if __name__ == "__main__":
    main()
