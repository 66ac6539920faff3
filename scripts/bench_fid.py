#!/usr/bin/env python
"""FID features (pytorch-fid's InceptionV3 up to the 2048-wide pool3 features) for one batch of 50 uint8 256^2 images
(fid_score.py's default --batch-size), seeded weights (oracle/fid_oracle.py weights with the BatchNorm statistics of
tests/golden/fid_inception.pt).

    python scripts/bench_fid.py [--rounds 7] [--reps 10]

Arms, in alternating rounds, each timed with CUDA events over --reps calls of the same batch on the device:
- fid.FIDInception.features from the device uint8 images (the preprocess and all 94 convs on this package's kernels,
  one CUDA graph replay per call);
- the oracle's torch module on cuDNN fp32 from the same bytes (ToTensor, F.interpolate and 2 x - 1 as torch ops on the
  device, as pytorch-fid runs them), with cudnn.allow_tf32 True (torch's default: what pytorch-fid runs) and False.
Reports images/s (median over rounds), the achieved algorithmic TFLOP/s (11.4 GFLOP per image, counted from the layer
shapes), and max |feature difference| of each cuDNN arm against this package's features.  Prints ONE JSON line with
the card's name, power limit and max SM clock.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from omnitokenizer_b200 import fid  # noqa: E402
from oracle import fid_oracle as fo  # noqa: E402
from scripts.bench_ingest import card  # noqa: E402

B, S = 50, 256


def flop_per_image() -> int:
    """2 x MACs of the 94 convolutions at a 299^2 input, from the layer shapes."""
    tot, hw = 0, (299, 299)

    def conv(c, src):
        nonlocal tot
        o = tuple(fid.out_size(n, k, c.s, p) for n, k, p in zip(src, c.k, c.p))
        tot += 2 * o[0] * o[1] * c.cout * c.cin * c.k[0] * c.k[1]
        return o

    for layer in fid.STEM:
        hw = conv(layer, hw) if isinstance(layer, fid.Conv) else tuple(
            fid.out_size(n, layer.k, layer.s, layer.p) for n in hw)
    for _, convs, pool, _ in fid.BLOCKS:
        shapes = {"x": hw, "p": hw}
        for c in convs:
            shapes[c.name] = conv(c, shapes[c.src])
        if pool.col is not None:
            hw = tuple(fid.out_size(n, pool.k, pool.s, pool.p) for n in hw)
    return tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_fid.py measures on a GPU"
    dev = torch.device("cuda:0")
    golden = torch.load(os.path.join(ROOT, "tests", "golden", "fid_inception.pt"))
    sd = fo.make_state_dict(golden["w_seed"])
    sd.update(golden["bn"])
    net = fid.FIDInception(sd, dev)
    sd_dev = {k: v.to(dev) for k, v in sd.items()}
    u8 = torch.randint(0, 256, (B, S, S, 3), generator=torch.Generator().manual_seed(1), dtype=torch.uint8).to(dev)

    def ours():
        return net.features(u8)

    def cudnn():
        with torch.no_grad():
            x = u8.permute(0, 3, 1, 2).contiguous().float().div(255)
            x = 2 * F.interpolate(x, size=(299, 299), mode="bilinear", align_corners=False) - 1
            return fo.forward(sd_dev, x)

    def arm(fn, tf32):
        torch.backends.cudnn.allow_tf32 = tf32
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        for _ in range(args.reps):
            out = fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / args.reps, out.clone()

    arms = {"omt_fid": (ours, True), "cudnn_tf32": (cudnn, True), "cudnn_fp32": (cudnn, False)}
    for _ in range(2):                                      # warm-up: the graph captured, cuDNN algorithms picked
        for fn, tf32 in arms.values():
            arm(fn, tf32)
    ms = {k: [] for k in arms}
    feats = {}
    for _ in range(args.rounds):
        for k, (fn, tf32) in arms.items():
            t, feats[k] = arm(fn, tf32)
            ms[k].append(t)
    torch.backends.cudnn.allow_tf32 = True
    flop = flop_per_image()
    med = {k: float(np.median(v)) for k, v in ms.items()}
    out = {
        "metric": "fid_features_images_per_s", "workload": f"{B} uint8 images {S}x{S} -> 299x299 pool3 features",
        "images_per_s": {k: round(B / (v * 1e-3), 1) for k, v in med.items()},
        "ms_per_batch": {k: round(v, 3) for k, v in med.items()},
        "ms_per_batch_range": {k: [round(min(v), 3), round(max(v), 3)] for k, v in ms.items()},
        "speedup_vs_cudnn_tf32": round(med["cudnn_tf32"] / med["omt_fid"], 2),
        "speedup_vs_cudnn_fp32": round(med["cudnn_fp32"] / med["omt_fid"], 2),
        "gflop_per_image": round(flop / 1e9, 2),
        "algorithmic_tflops_per_s": {k: round(B * flop / (v * 1e-3) / 1e12, 1) for k, v in med.items()},
        "max_abs_feature": round(float(feats["omt_fid"].abs().max()), 4),
        "max_dfeature_vs_cudnn_tf32": float((feats["omt_fid"] - feats["cudnn_tf32"]).abs().max()),
        "max_dfeature_vs_cudnn_fp32": float((feats["omt_fid"] - feats["cudnn_fp32"]).abs().max()),
        "rounds": args.rounds, "reps": args.reps,
        "card": card(),
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
