#!/usr/bin/env python
"""Baseline JPEG decoding of ImageNet-like files on the device against Pillow on the host.

    python scripts/bench_jpeg_decode.py [--reps 20] [--rounds 5]

Files: seeded 500 x 375 smooth images with a little noise (oracle/jpeg_oracle.py content "smooth"), saved by Pillow at
quality 90, 4:2:0, batches of 64 and 256.
- device: jpeg.decode_u8 (staging, omt_jpeg_decode_u8, status read back), host clock around --reps calls that end in a
  synchronise, median of --rounds; images/s and compressed MB/s; per-stage CUDA-event times and the synchronisation's
  launch count (omt_jpeg_decode_u8_timed);
- host: Pillow's Image.open(BytesIO(f)).convert("RGB") of the same files on 1 process and on os.cpu_count() processes;
- whether every decoded byte equals Pillow's;
- a 256^2 eval batch (--encode-batch files, the canonical model with seeded weights, layout.image_resize(256)):
  model.encode_jpeg_u8 of the files against Pillow's decode on one host thread + model.encode_images_u8, alternating,
  host clock around synchronised calls, median of --rounds; whether the codes agree.
Prints ONE JSON line with the card's name, power limit and max SM clock.
"""
import argparse
import io
import json
import os
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from omnitokenizer_b200 import jpeg  # noqa: E402
from oracle import jpeg_decode_oracle as D  # noqa: E402
from scripts.bench_ingest import card  # noqa: E402


def _pillow(files):
    from PIL import Image
    return [np.asarray(Image.open(io.BytesIO(f)).convert("RGB")) for f in files]


def _median_s(fn, rounds):
    ts = []
    for _ in range(rounds):
        t = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--encode-batch", type=int, default=32)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_jpeg_decode.py needs a CUDA device")
    dev = torch.device("cuda:0")
    res = {"card": card()}
    cpus = os.cpu_count() or 1
    with ProcessPoolExecutor(cpus) as pool:
        for B in (64, 256):
            files = [D.fixture(375, 500, "4:2:0", 90, "smooth", 5000 + i) for i in range(B)]
            mb = sum(map(len, files)) / 1e6
            jpeg.decode_u8(files, dev)
            torch.cuda.synchronize()

            def device():
                for _ in range(a.reps):
                    jpeg.decode_u8(files, dev)
                torch.cuda.synchronize()
            t_dev = _median_s(device, a.rounds) / a.reps
            stages = {}
            jpeg.decode_u8(files, dev, timings=stages)
            t_pil1 = _median_s(lambda: _pillow(files), max(1, a.rounds // 2))
            chunks = [files[i::cpus] for i in range(cpus)]
            list(pool.map(_pillow, chunks))
            t_pool = _median_s(lambda: list(pool.map(_pillow, chunks)), a.rounds)
            got = jpeg.decode_u8(files, dev)
            same = all(np.array_equal(g.cpu().numpy(), p) for g, p in zip(got, _pillow(files)))
            res[f"B{B}"] = {"compressed_MB": round(mb, 3), "device_ms": round(1e3 * t_dev, 3),
                            "device_images_per_s": round(B / t_dev, 1), "device_MB_per_s": round(mb / t_dev, 1),
                            "stages_ms": {k: round(v, 4) if isinstance(v, float) else v for k, v in stages.items()},
                            "pillow_1proc_ms": round(1e3 * t_pil1, 2), "pillow_1proc_images_per_s": round(B / t_pil1, 1),
                            f"pillow_{cpus}proc_ms": round(1e3 * t_pool, 2),
                            f"pillow_{cpus}proc_images_per_s": round(B / t_pool, 1), "bytes_equal": same}
    res["encode_256"] = encode_batch(dev, a.encode_batch, a.rounds)
    print(json.dumps(res))


def encode_batch(dev, B, rounds):
    import omnitokenizer_b200 as ob
    from omnitokenizer_b200 import layout as L
    from oracle import omni_oracle as oo
    from oracle import weights as W
    args = ob.canonical_args()
    m = ob.OmniTokenizer_VQGAN(args)
    m.load_state_dict(W.make_state_dict(oo.Config.from_args(args), 0), strict=False)
    m.codebook._need_init = False
    m = m.to(dev).eval()
    rz = L.image_resize(256)
    files = [D.fixture(375, 500, "4:2:0", 90, "smooth", 7000 + i) for i in range(B)]

    def host():
        torch.manual_seed(0)
        out = m.encode_images_u8([torch.from_numpy(a.copy()) for a in _pillow(files)], rz)
        torch.cuda.synchronize()
        return out

    def device():
        torch.manual_seed(0)
        out = m.encode_jpeg_u8(files, rz)
        torch.cuda.synchronize()
        return out
    same = torch.equal(host(), device()) and torch.equal(host(), device())      # warms both (eager, then graph)
    th, td = [], []
    for _ in range(rounds):
        for fn, ts in ((host, th), (device, td)):
            t = time.perf_counter()
            fn()
            ts.append(time.perf_counter() - t)
    return {"files": B, "host_decode_plus_encode_images_u8_ms": round(1e3 * float(np.median(th)), 2),
            "encode_jpeg_u8_ms": round(1e3 * float(np.median(td)), 2), "codes_equal": same}


if __name__ == "__main__":
    main()
