#!/usr/bin/env python
"""The video-metric suite's calculate_fvd on gFVD-shaped work: 2 x --clips clips of --frames frames at --size^2 (both
sides uint8), seeded I3D weights, every prefix t = 10 ... frames, both methods.

    python scripts/bench_fvd_suite.py [--clips 256] [--frames 17] [--size 128] [--rounds 2]

Arms, in alternating rounds, each ending in a synchronise:
- (a) the suite's way: the clips as fp32 (B, T, 3, H, W) on the host, each prefix's preprocess on the host (the
  oracle's restatement of the method's preprocess_single, bit for bit the reference's; torch's default threads), the
  network input to the device in chunks of 10 clips (get_feats's bs) and I3D as torch ops on the GPU (cuDNN, TF32
  allowed: torch's defaults), the features to the host;
- (b) quality.calculate_fvd from the device uint8 clips.
Reports ms per full prefix sweep of each arm, the I3D device time of (b) (CUDA events around every features call,
preprocess included), its algorithmic TFLOP/s (bench_fvd.work's layer shapes), max |feature difference| of (a) and (b)
at the longest prefix, and the card's name, power limit and max SM clock.  Prints ONE JSON line.
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from omnitokenizer_b200 import fvd, quality  # noqa: E402
from oracle import fvd_suite_oracle as so  # noqa: E402
from oracle import i3d_oracle as io  # noqa: E402
from scripts.bench_fvd import work  # noqa: E402
from scripts.bench_ingest import card  # noqa: E402

DEV = torch.device("cuda:0")


def seeded_sd():
    g = torch.load(os.path.join(ROOT, "tests", "golden", "fvd_i3d.pt"))
    sd = io.make_state_dict(g["w_seed"])
    sd.update(g["bn"])
    return sd


def suite_arm(sd, eps, method, f32_host, T):
    """The suite's calculate_fvd loop with torch I3D on the GPU; returns the features of the last prefix."""
    pre = so.preprocess_styleganv if method == "styleganv" else so.preprocess_videogpt
    sd_dev = {k: v.to(DEV) for k, v in sd.items()}
    feats = None
    for t in range(10, T + 1):
        feats = []
        for side in f32_host:
            x = pre(side, t)
            f = [io.forward(sd_dev, x[i:i + 10].to(DEV), eps=eps).cpu() for i in range(0, x.shape[0], 10)]
            feats.append(torch.cat(f).double())
        if method == "styleganv":
            quality.frechet_distance_styleganv(feats[0].numpy(), feats[1].numpy())
        else:
            quality.frechet_distance_videogpt(feats[0], feats[1])
    return feats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=256)
    ap.add_argument("--frames", type=int, default=17)
    ap.add_argument("--size", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fvd_suite.py needs a GPU")
    B, T, S = args.clips, args.frames, args.size
    g = torch.Generator().manual_seed(0)
    sides_u8 = [torch.randint(0, 256, (B, T, S, S, 3), generator=g, dtype=torch.uint8) for _ in range(2)]
    f32_host = [u.float().permute(0, 1, 4, 2, 3).contiguous() / 255. for u in sides_u8]
    dev_u8 = [u.to(DEV) for u in sides_u8]
    sd = seeded_sd()
    nets = {"videogpt": fvd.I3D(sd, DEV), "styleganv": fvd.I3D(sd, DEV, variant="styleganv")}
    eps = {m: fvd.VARIANT_EPS[m] for m in nets}
    res = {"clips": B, "frames": T, "size": S, "prefixes": T - 9}
    algo = sum(2 * work(B, t)[0] for t in range(10, T + 1))
    for method, net in nets.items():
        times = {"suite": [], "ours": []}
        i3d_ms, events = [], []
        orig = net.features

        def timed(clips, t):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = orig(clips, t)
            e1.record()
            events.append((e0, e1))
            return out

        net.features = timed
        quality.calculate_fvd(dev_u8[0], dev_u8[1], "cuda", method, i3d=net)      # warm: workspaces, graphs
        for _ in range(args.rounds):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ref = suite_arm(sd, eps[method], method, f32_host, T)
            torch.cuda.synchronize()
            times["suite"].append((time.perf_counter() - t0) * 1e3)
            events.clear()
            t0 = time.perf_counter()
            quality.calculate_fvd(dev_u8[0], dev_u8[1], "cuda", method, i3d=net)
            torch.cuda.synchronize()
            times["ours"].append((time.perf_counter() - t0) * 1e3)
            i3d_ms.append(sum(a.elapsed_time(b) for a, b in events))
            print(f"{method}: suite {times['suite'][-1]:.0f} ms, ours {times['ours'][-1]:.0f} ms", file=sys.stderr)
        del net.features
        ours = [net.features(fvd.SuiteClips(u, fvd.FORM_U8), T).double().cpu() for u in dev_u8]
        diff = max(float((a - b).abs().max()) for a, b in zip(ours, ref))
        res[method] = {"suite_ms_per_sweep": min(times["suite"]), "ours_ms_per_sweep": min(times["ours"]),
                       "ours_i3d_device_ms": min(i3d_ms), "ours_algo_tflops": algo / (min(i3d_ms) * 1e-3) / 1e12,
                       "speedup": min(times["suite"]) / min(times["ours"]), "max_feature_diff": diff,
                       "max_abs_feature": float(ours[0].abs().max())}
    res["card"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
