#!/usr/bin/env python
"""The JPEG save and reload vqgan_eval.py pays for each side of every image batch on a .jpg / .JPEG dataset, on the
device and on the host.

    python scripts/bench_jpeg.py [--reps 50] [--rounds 5]

Batches: 64 x 256^2 (ImageNet at --resolution 256) and 50 x 128^2, seeded smooth images with a little noise
(oracle/jpeg_oracle.py content "smooth"), quality 75.
- device: jpeg.roundtrip_u8 (omt_jpeg_roundtrip_u8, two launches), CUDA events over --reps calls, median of --rounds;
- host: Pillow's save(BytesIO, "JPEG") + Image.open(...).convert("RGB") of every image, one thread, median of --rounds.
Checks that both give the same bytes.  Prints ONE JSON line with the card's name, power limit and max SM clock.
"""
import argparse
import io
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from omnitokenizer_b200 import jpeg  # noqa: E402
from oracle import jpeg_oracle as J  # noqa: E402
from scripts.bench_ingest import card  # noqa: E402

BATCHES = [(64, 256), (50, 128)]


def pillow_batch(images: np.ndarray) -> np.ndarray:
    from PIL import Image
    out = []
    for a in images:
        f = io.BytesIO()
        Image.fromarray(a).save(f, "JPEG", quality=jpeg.DEFAULT_QUALITY)
        f.seek(0)
        out.append(np.asarray(Image.open(f).convert("RGB")))
    return np.stack(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_jpeg.py measures on a GPU"
    dev = torch.device("cuda:0")
    results = []
    for B, S in BATCHES:
        host = np.stack([J.content("smooth", S, S, 100 + i) for i in range(B)])
        x = torch.from_numpy(host).to(dev)
        for _ in range(3):                                     # warm-up: module load, scratch allocation
            y = jpeg.roundtrip_u8(x)
        torch.cuda.synchronize()
        dev_ms = []
        for _ in range(args.rounds):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.reps):
                jpeg.roundtrip_u8(x)
            b.record()
            torch.cuda.synchronize()
            dev_ms.append(a.elapsed_time(b) / args.reps)
        host_ms = []
        want = None
        for _ in range(args.rounds):
            t0 = time.perf_counter()
            want = pillow_batch(host)
            host_ms.append((time.perf_counter() - t0) * 1e3)
        same = bool(np.array_equal(y.cpu().numpy(), want))
        pixels = B * S * S
        results.append({
            "batch": f"{B}x{S}x{S}", "device_ms": round(float(np.median(dev_ms)), 4),
            "device_ms_spread": [round(min(dev_ms), 4), round(max(dev_ms), 4)],
            "host_pillow_ms": round(float(np.median(host_ms)), 2),
            # bytes the two launches must move at least: src and dst (3 B / pixel each), the planes written and read
            "device_GBps": round(pixels * (3 + 3 + 2 * 1.5) / (float(np.median(dev_ms)) * 1e-3) / 1e9, 1),
            "bytes_equal_pillow": same})
    print(json.dumps({"metric": "jpeg_roundtrip_ms_per_batch", "quality": jpeg.DEFAULT_QUALITY, "reps": args.reps,
                      "rounds": args.rounds, "results": results, "host_threads": 1, "card": card()}))


if __name__ == "__main__":
    main()
