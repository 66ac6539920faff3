"""Per-frame reconstruction metrics of one cfg-3 eval batch (8 clips x 17 frames of 256^2, uint8 on the device):
quality.frame_metrics with PSNR + SSIM alone and with the VGG LPIPS (seeded weights), against the oracle's LPIPS as a
torch CUDA fp32 module (cuDNN, TF32 off and on) in the same process, and numpy / cv2 PSNR + SSIM on the host (the
suite's own functions' arithmetic, a few frames, scaled).  CUDA-event timing, alternating rounds; one JSON line with
the card, power limit and max SM clock.

    python scripts/bench_quality.py [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from omnitokenizer_b200 import quality  # noqa: E402
from oracle import quality_oracle as qo  # noqa: E402

B, T, H, W = 8, 17, 256, 256
VGG_GFLOP = 2 * sum(9 * ci * co * (H * W) / 4 ** s for s, convs in enumerate(qo.VGG_SLICES)
                    for _, ci, co in convs) / 1e9          # per image, from the shapes


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def timed(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    real = torch.randint(0, 250, (B, T, H, W, 3), generator=g, dtype=torch.uint8)
    fake = (real.to(torch.int16) + torch.randint(-20, 21, real.shape, generator=g, dtype=torch.int16)).clamp(0, 255)
    real, fake = real.to(dev), fake.to(torch.uint8).to(dev)
    sd = qo.make_state_dict(5)
    net = quality.LPIPS(sd, dev)
    sd_dev = {k: v.to(dev) for k, v in sd.items()}
    a01 = qo.to01(real.flatten(0, 1))
    b01 = qo.to01(fake.flatten(0, 1))
    P = B * T

    def ours_plain():
        quality.frame_metrics(real, fake)

    def ours_lpips():
        quality.frame_metrics(real, fake, net)

    def torch_lpips(tf32):
        def run():
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32
            with torch.no_grad():
                for i in range(0, P, 8):           # the oracle module in batches of 8 pairs
                    qo.lpips(sd_dev, a01[i:i + 8], b01[i:i + 8])
        return run

    for f in (ours_plain, ours_lpips, ours_lpips, ours_lpips, torch_lpips(False), torch_lpips(True)):
        f()                                          # warm-up: eager, capture, replay; cuDNN algorithm choice
    res = {"plain": [], "lpips": [], "torch_fp32": [], "torch_tf32": []}
    for _ in range(args.rounds):
        res["plain"].append(timed(ours_plain, args.reps * 4))
        res["lpips"].append(timed(ours_lpips, args.reps))
        res["torch_fp32"].append(timed(torch_lpips(False), 1))
        res["torch_tf32"].append(timed(torch_lpips(True), 1))
    torch.backends.cudnn.allow_tf32 = True
    ms = {k: float(np.median(v)) for k, v in res.items()}
    # accuracy of this run's LPIPS against the fp32 oracle on the device with TF32 off
    torch.backends.cudnn.allow_tf32 = False
    with torch.no_grad():
        ref = torch.cat([qo.lpips(sd_dev, a01[i:i + 8], b01[i:i + 8]) for i in range(0, P, 8)])
    torch.backends.cudnn.allow_tf32 = True
    got = quality.frame_metrics(real, fake, net)[2].flatten()
    lp_rel = float(((got - ref).abs() / ref.abs()).max())
    # host: the suite's numpy / cv2 arithmetic on a few frames (float64 inputs), scaled to the batch
    import cv2
    win = np.outer(cv2.getGaussianKernel(11, 1.5), cv2.getGaussianKernel(11, 1.5).T)
    n_host = 8
    ah = qo.to01(real[0, :n_host].cpu()).double().numpy()
    bh = qo.to01(fake[0, :n_host].cpu()).double().numpy()
    t0 = time.perf_counter()
    for i in range(n_host):
        qo.psnr(ah[i], bh[i])
        for c in range(3):
            x, y = ah[i, c], bh[i, c]
            for z in (x, y, x * x, y * y, x * y):
                cv2.filter2D(z, -1, win)
    host_ms = (time.perf_counter() - t0) * 1e3 / n_host * P
    out = {
        "card": card(), "batch": f"{B}x{T}x{H}x{W}",
        "frame_pairs_per_s": {"psnr_ssim": P / ms["plain"] * 1e3, "psnr_ssim_lpips": P / ms["lpips"] * 1e3,
                              "torch_lpips_fp32": P / ms["torch_fp32"] * 1e3,
                              "torch_lpips_tf32": P / ms["torch_tf32"] * 1e3,
                              "host_cv2_psnr_ssim": P / host_ms * 1e3},
        "ms_per_batch": {**ms, "host_cv2_psnr_ssim": host_ms},
        "lpips_tflops": 2 * P * VGG_GFLOP / ms["lpips"],
        "vgg_gflop_per_image": VGG_GFLOP,
        "lpips_rel_vs_fp32_torch": lp_rel,
        "rounds_ms": res,
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
