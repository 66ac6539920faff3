#!/usr/bin/env python
"""Image input side: the loaders' Pillow resize (+ flip) on the host, or on the device with omt_resample_u8.

    python scripts/bench_resize_ingest.py [--batch 64] [--res 256] [--steps 10] [--reps 200]

On a seeded batch of decoded uint8 images of ImageNet-like sizes (mostly 500 x 375 / 375 x 500 / 500 x 333, some larger):
- host: ms per batch of the DiT loader's transform (Diffusion/DiT/train.py:192-198 with the OmniTokenizer VAE:
  torchvision Resize((res, res)) bilinear + RandomHorizontalFlip on the PIL images, then the uint8 arrays stacked), on
  1 thread and on a pool of os.cpu_count() threads (Pillow releases the GIL while it resizes); and of the bicubic
  Resize of ImageDataset (OmniTokenizer/data.py:93-99) on 1 thread;
- stage: host ms of Engine.stage_images_u8 (descriptors, coefficient tables, source bytes into pinned memory + async copy);
- h2d: bytes of the source images against the resized batch;
- kernel: device time of omt_resample_u8 (CUDA events over --reps launches after a warm-up), bilinear and bicubic;
- e2e: images/s of the DiT latent encode, "host": host transform (thread pool) -> pinned stack -> encode_u8 -> latents,
  against "device": encode_images_u8 -> latents, alternating, each step ending in a synchronise; the latents of both
  under the same seed are compared bit for bit.
Prints ONE JSON line with the card's name and power limit.
"""
import argparse
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.bench_ingest import card, ev_ms  # noqa: E402

# (H, W) of decoded ImageNet-like photos and their weights in the batch
PHOTO_SIZES = [((375, 500), 5), ((500, 375), 2), ((333, 500), 2), ((500, 333), 1), ((500, 500), 1), ((480, 640), 1),
               ((768, 1024), 1)]


def sources(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    sizes = [s for s, w in PHOTO_SIZES for _ in range(w)]
    pick = torch.randint(0, len(sizes), (n,), generator=g).tolist()
    return [torch.randint(0, 256, sizes[k] + (3,), generator=g, dtype=torch.uint8) for k in pick]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--res", type=int, default=256)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=200)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_resize_ingest.py measures on the GPU; there is no CPU mode"
    from PIL import Image
    from torchvision import transforms
    from torchvision.transforms import InterpolationMode

    import omnitokenizer_b200 as ob
    from omnitokenizer_b200 import _cabi, consumers as C
    from omnitokenizer_b200 import layout as L

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    B, res = args.batch, args.res
    imgs = sources(B)
    pils = [Image.fromarray(im.numpy()) for im in imgs]
    out = {"card": card(), "math": os.environ.get("OMT_MATH", "f16x3"), "host_cpus": os.cpu_count(), "batch": B, "res": res,
           "source_sizes": sorted({tuple(im.shape[:2]) for im in imgs})}

    dit_tf = transforms.Compose([transforms.Resize((res, res)), transforms.RandomHorizontalFlip()])
    img_tf = transforms.Compose([transforms.Resize((res, res), interpolation=InterpolationMode.BICUBIC)])
    pool = ThreadPoolExecutor(os.cpu_count())

    def host_batch(tf, threads, dst=None):
        one = lambda p: np.array(tf(p))          # noqa: E731  (a copy, as ToTensor's np.array(pic, copy=True))
        arrs = list(pool.map(one, pils)) if threads > 1 else [one(p) for p in pils]
        return torch.stack([torch.from_numpy(a) for a in arrs], out=dst)

    # ---- host transform
    host = {}
    for label, tf, threads in (("dit_1_thread", dit_tf, 1), ("dit_pool", dit_tf, os.cpu_count()),
                               ("image_bicubic_1_thread", img_tf, 1)):
        host_batch(tf, threads)
        t0 = time.perf_counter()
        n = 3
        for _ in range(n):
            host_batch(tf, threads)
        host[label] = {"threads": threads, "ms_per_batch": round((time.perf_counter() - t0) * 1e3 / n, 2)}
    out["host"] = host

    # ---- model (VAE, as DiT uses it), staging, H2D bytes, kernel time
    m = ob.OmniTokenizer_VQGAN(ob.canonical_args(["--use_vae", "--resolution", str(res)]))
    m.codebook._need_init = False
    m = m.to(dev).eval()
    eng = m.prepare().engine()
    resized = torch.empty(B, res, res, 3, dtype=torch.uint8, device=dev)
    kern = {}
    for name, rz in (("bilinear_dit", L.dit_resize(res)), ("bicubic_image", L.image_resize(res))):
        torch.manual_seed(1)
        params = L.resize_params(B, rz)
        eng.stage_images_u8(imgs, rz, params)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(5):
            a = eng.stage_images_u8(imgs, rz, params)
        torch.cuda.synchronize()
        stage_ms = (time.perf_counter() - t0) * 1e3 / 5
        launch = lambda: _cabi.call("omt_resample_u8", *a, resized)         # noqa: E731
        us = [round(ev_ms(launch, args.reps) * 1e3, 1) for _ in range(2)]
        want = torch.stack([L.resize_u8(im, rz, p) for im, p in zip(imgs[:4], params[:4])])
        kern[name] = {"kernel_us": us, "stage_ms": round(stage_ms, 2),
                      "first4_equal_host": bool(torch.equal(resized[:4].cpu(), want))}
        out["h2d"] = {"source_bytes": int(a[1]), "resized_bytes": B * res * res * 3,
                      "ratio": round(a[1] / (B * res * res * 3), 2)}
    out["kernel"] = kern

    # ---- e2e DiT latent encode, alternating
    pinned = torch.empty(B, res, res, 3, dtype=torch.uint8).pin_memory()

    def host_step():
        x = host_batch(dit_tf, os.cpu_count(), pinned)
        return C.dit_encode_latents_u8(m, x.to(dev, non_blocking=True), C.IMAGE_NORM)

    def dev_step():
        return C.dit_encode_latents_images_u8(m, imgs, res)

    e2e = {}
    for rnd in range(2):
        for name, step in (("host", host_step), ("device", dev_step)):
            for _ in range(3):
                step()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                step()
                torch.cuda.synchronize()
            e2e.setdefault(name, []).append(round(B * args.steps / (time.perf_counter() - t0), 1))
    out["e2e_images_per_s"] = e2e
    # same seed, same flips and noise: the latents of the two paths (host transform sequential, in the loader's order)
    torch.manual_seed(7)
    x = host_batch(dit_tf, 1)
    z_host = C.dit_encode_latents_u8(m, x.to(dev), C.IMAGE_NORM)
    torch.manual_seed(7)
    z_dev = dev_step()
    out["latents_equal"] = bool(torch.equal(z_host, z_dev))
    pool.shutdown()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
