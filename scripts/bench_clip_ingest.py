#!/usr/bin/env python
"""Video input side: the Latte loaders' fp32 transform on the host, or on the device with omt_resample_clips.

    python scripts/bench_clip_ingest.py [--steps 10] [--reps 200]

Two batches of decoded uint8 clips (F, H, W, 3), 17 frames each, to 256^2 with UCFCenterCropVideo (layout.ucf_clip_resize,
Latte's configs/ucf101/ucf101_train_omnitokenizer.yaml: local_batch_size 5, num_frames 17, image_size 256):
- "ucf": 5 clips at UCF-101's 240 x 320;
- "mixed": 5 clips of different sizes (240 x 320 to 720 x 1280).
Per batch it reports:
- host: ms of the loader's Compose (ToTensorVideo, RandomHorizontalFlipVideo, UCFCenterCropVideo, Normalize; torch on one
  thread, as in a DataLoader worker) on 1 thread and on a pool of os.cpu_count() threads, one clip per task;
- stage: host ms of Engine.stage_clips_u8 (descriptors, axis tables, source bytes into pinned memory + async copy);
- h2d: bytes of the decoded clips against the fp32 clips the host path copies;
- kernel: device time of omt_resample_clips (CUDA events over --reps launches after a warm-up);
- e2e: clips/s of latte_encode_latents, "host": pool transform -> pinned stack -> latte_encode_latents, against
  "device": latte_encode_latents_clips_u8, alternating, each step ending in a synchronise; the latents of both under
  the same seeds are compared bit for bit.
Prints ONE JSON line with the card's name and power limit.
"""
import argparse
import json
import os
import random
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import torch
import torch.nn.functional as Fn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.bench_ingest import card, ev_ms  # noqa: E402

F, S = 17, 256
BATCHES = {"ucf": [(240, 320)] * 5, "mixed": [(240, 320), (360, 480), (720, 1280), (256, 340), (480, 640)]}


def sources(sizes, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 256, (F, h, w, 3), generator=g, dtype=torch.uint8) for h, w in sizes]


def host_clip(clip, flip):
    """Latte's ucf101 Compose (datasets/__init__.py, video_transforms.py) on a read_video-style (F, 3, H, W) view."""
    x = clip.permute(0, 3, 1, 2).float() / 255.0
    if flip:
        x = x.flip(-1)
    x = Fn.interpolate(x, scale_factor=S / min(x.shape[-2:]), mode="bilinear", align_corners=False)
    h, w = x.shape[-2:]
    i, j = int(round((h - S) / 2.0)), int(round((w - S) / 2.0))
    x = x[..., i:i + S, j:j + S]
    return x.sub_(torch.tensor([0.5] * 3).view(-1, 1, 1)).div_(torch.tensor([0.5] * 3).view(-1, 1, 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=200)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_clip_ingest.py measures on the GPU; there is no CPU mode"
    import omnitokenizer_b200 as ob
    from omnitokenizer_b200 import _cabi, consumers as C
    from omnitokenizer_b200 import layout as L

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    torch.set_num_threads(1)                  # the loader's workers run torch on one thread
    rz = L.ucf_clip_resize(S)
    pool = ThreadPoolExecutor(os.cpu_count())
    out = {"card": card(), "math": os.environ.get("OMT_MATH", "f16x3"), "host_cpus": os.cpu_count(), "frames": F,
           "size": S, "cpu_capability": torch.backends.cpu.get_cpu_capability()}

    m = ob.OmniTokenizer_VQGAN(ob.canonical_args(["--use_vae", "--resolution", str(S)]))
    m.codebook._need_init = False
    m = m.to(dev).eval()
    eng = m.prepare().engine()

    def host_batch(clips, flips, threads, dst=None):
        one = lambda cf: host_clip(*cf)       # noqa: E731
        xs = list(pool.map(one, zip(clips, flips))) if threads > 1 else [one(cf) for cf in zip(clips, flips)]
        return torch.stack(xs, out=dst)

    for name, sizes in BATCHES.items():
        clips = sources(sizes, seed=len(name))
        B = len(clips)
        res = {"sources": sorted(set(sizes))}
        random.seed(1)
        flips = L.clip_params(B, rz)
        host = {}
        for label, threads in (("1_thread", 1), ("pool", os.cpu_count())):
            host_batch(clips, flips, threads)
            t0 = time.perf_counter()
            for _ in range(3):
                host_batch(clips, flips, threads)
            host[label] = {"threads": threads, "ms_per_batch": round((time.perf_counter() - t0) * 1e3 / 3, 2)}
        res["host"] = host

        eng.stage_clips_u8(clips, rz, flips)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(5):
            a, shape = eng.stage_clips_u8(clips, rz, flips)
        torch.cuda.synchronize()
        res["stage_ms"] = round((time.perf_counter() - t0) * 1e3 / 5, 2)
        x = torch.empty(B, 3, F, S, S, device=dev)
        lut = eng._table(("clipnorm", C.LATTE_NORM), lambda: L.clip_norm_table(C.LATTE_NORM))
        launch = lambda: _cabi.call("omt_resample_clips", *a, lut, *shape, x)       # noqa: E731
        res["kernel_us"] = [round(ev_ms(launch, args.reps) * 1e3, 1) for _ in range(2)]
        res["kernel_equal_host"] = bool(torch.equal(x.cpu().transpose(1, 2), host_batch(clips, flips, 1)))
        res["h2d"] = {"source_bytes": int(a[1]), "fp32_clip_bytes": B * F * 3 * S * S * 4,
                      "ratio": round(B * F * 3 * S * S * 4 / a[1], 2)}

        pinned = torch.empty(B, F, 3, S, S).pin_memory()

        def host_step():
            fl = L.clip_params(B, rz)
            return C.latte_encode_latents(m, host_batch(clips, fl, os.cpu_count(), pinned).to(dev, non_blocking=True))

        def dev_step():
            return C.latte_encode_latents_clips_u8(m, clips, rz)

        e2e = {}
        for rnd in range(2):
            for label, step in (("host", host_step), ("device", dev_step)):
                for _ in range(3):
                    step()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(args.steps):
                    step()
                    torch.cuda.synchronize()
                e2e.setdefault(label, []).append(round(B * args.steps / (time.perf_counter() - t0), 2))
        res["e2e_clips_per_s"] = e2e
        random.seed(7)
        torch.manual_seed(7)
        z_host = host_step()
        random.seed(7)
        torch.manual_seed(7)
        z_dev = dev_step()
        res["latents_equal"] = bool(torch.equal(z_host, z_dev))
        out[name] = res
    pool.shutdown()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
