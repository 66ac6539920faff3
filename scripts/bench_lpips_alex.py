"""The suite's calculate_lpips (the lpips package's AlexNet, spatial=True; seeded weights) on two workloads: the demo's
8 videos x 30 frames of 64^2 and one cfg-3 eval batch, 8 x 17 frames of 256^2.  quality.calculate_lpips is timed on fp32
host videos (the upload included), fp32 device videos and uint8 device frames; in the same process, the suite's own
per-frame loop (the oracle module on the GPU, torch's default cuDNN settings, one forward and one host sync per frame)
and one batched eager forward of the oracle module in strict fp32 and in TF32, from the host videos and from the same
videos already on the device.  CUDA events around each whole call, medians of alternating rounds.  Each AlexNet conv
is also timed alone at the workload's shape: omt_conv3d against cuDNN's conv2d in strict fp32 and in TF32.  The
largest per-frame difference of each eager variant from quality.calculate_lpips is printed as information (the suite's
TF32 values are not the bar).  One JSON line per workload with the card, power limit and max SM clock.

    python scripts/bench_lpips_alex.py [--rounds 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from omnitokenizer_b200 import quality  # noqa: E402
from oracle import lpips_alex_oracle as ao  # noqa: E402

WORKLOADS = {"demo_8x30x64": (8, 30, 64, 64), "cfg3_8x17x256": (8, 17, 256, 256)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def timed(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    out = fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e), out


def conv_layers(model, net, B2, H, W, reps):
    """Each AlexNet conv alone at the workload's 2 B T images, inputs already on the device: omt_conv3d (the packed
    3xTF32 conv the trunk launches, channels-last input) against cuDNN's F.conv2d (NCHW, as the lpips module runs it)
    in strict fp32 and in TF32.  ms per launch over `reps` launches, CUDA events."""
    default_tf32 = torch.backends.cudnn.allow_tf32
    g = torch.Generator().manual_seed(3)
    out, h, w = {}, H, W
    for c, u in zip(quality.ALEX, model.convs):
        if c.pool:
            h, w = (h - 3) // 2 + 1, (w - 3) // 2 + 1
        ho, wo = (h + 2 * c.pad - c.k) // c.stride + 1, (w + 2 * c.pad - c.k) // c.stride + 1
        x = torch.rand(B2, c.cin, h, w, generator=g).to("cuda")
        cs = 4 if c.cin == 3 else c.cin
        x_cl = torch.zeros(B2, h, w, cs, device="cuda")
        x_cl[..., :c.cin] = x.permute(0, 2, 3, 1)
        y = torch.empty(B2, ho, wo, c.cout, device="cuda")
        ours = u.launch(x_cl, B2, (1, h, w), (0, c.pad, c.pad), (1, ho, wo), y)
        conv = net.features[c.idx]
        row = {}
        for arm, fn, tf32 in (("omt_conv3d", ours, False), ("cudnn_fp32", lambda: conv(x), False),
                              ("cudnn_tf32", lambda: conv(x), True)):
            torch.backends.cudnn.allow_tf32 = tf32
            try:
                with torch.no_grad():
                    for _ in range(3):
                        fn()
                    row[arm] = round(timed(lambda: [fn() for _ in range(reps)])[0] / reps, 4)
            finally:
                torch.backends.cudnn.allow_tf32 = default_tf32
        out[f"conv{c.idx}_{c.cin}to{c.cout}_k{c.k}s{c.stride}_{h}x{w}"] = row
        h, w = ho, wo
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    sd = ao.make_state_dict(11)
    model = quality.AlexLPIPS(sd, dev)
    net = ao.AlexLPIPSOracle(sd).eval().to(dev)
    net.record = None                            # the suite's loop syncs once per frame by itself; no second sync
    default_tf32 = torch.backends.cudnn.allow_tf32

    def eager(v1, v2, tf32):
        """One batched forward of the lpips module and the per-frame means; v1, v2 host or device (B, T, 3, H, W)."""
        torch.backends.cudnn.allow_tf32 = tf32
        try:
            with torch.no_grad():
                a, b = (ao.trans(v.to(dev)).flatten(0, 1) for v in (v1, v2))
                return net.forward(a, b).mean((1, 2, 3)).view(v1.shape[:2])
        finally:
            torch.backends.cudnn.allow_tf32 = default_tf32

    def suite(v1, v2):
        with torch.no_grad():
            return ao.suite_loop(net, v1, v2, dev)

    for name, (B, T, H, W) in WORKLOADS.items():
        v1, v2 = ao.videos((B, T, 3, H, W, "bytes", 1))
        d1, d2 = v1.to(dev), v2.to(dev)          # uploaded once, outside every timed region
        u1, u2 = ao.to_u8(v1).to(dev), ao.to_u8(v2).to(dev)
        # *_host arms include the upload of both fp32 sides (pageable host memory); *_device arms start from frames
        # already on the device, so calculate_lpips_f32_device against eager_device_* compares the networks
        arms = {
            "calculate_lpips_f32_host": lambda: quality.calculate_lpips(v1, v2, dev, model),
            "calculate_lpips_f32_device": lambda: quality.calculate_lpips(d1, d2, dev, model),
            "calculate_lpips_u8_device": lambda: quality.calculate_lpips(u1, u2, dev, model),
            "suite_loop_cudnn_default": lambda: suite(v1, v2),
            "eager_host_fp32": lambda: eager(v1, v2, False),
            "eager_host_tf32": lambda: eager(v1, v2, True),
            "eager_device_fp32": lambda: eager(d1, d2, False),
            "eager_device_tf32": lambda: eager(d1, d2, True),
        }
        for fn in arms.values():                 # warm-up: modules, cuDNN algorithms, workspaces and CUDA graphs
            for _ in range(3):
                fn()
        times = {k: [] for k in arms}
        for r in range(args.rounds):
            order = list(arms) if r % 2 == 0 else list(arms)[::-1]
            for k in order:
                times[k].append(timed(arms[k])[0])
        ours = quality.lpips_alex_frames(v1, v2, dev, model).double().cpu()
        assert torch.equal(ours, quality.lpips_alex_frames(u1, u2, dev, model).double().cpu())
        assert torch.equal(ours, quality.lpips_alex_frames(d1, d2, dev, model).double().cpu())
        diffs = {}
        for k, fn in (("suite_loop_cudnn_default", lambda: suite(v1, v2)),
                      ("eager_fp32", lambda: eager(d1, d2, False)),
                      ("eager_tf32", lambda: eager(d1, d2, True))):
            ref = fn().double().cpu()
            diffs[k] = float(((ref - ours).abs() / ours.abs()).max())
        res = {"workload": name, "frames": B * T, "card": card(), "rounds": args.rounds,
               "ms_median": {k: round(statistics.median(v), 3) for k, v in times.items()},
               "ms_min": {k: round(min(v), 3) for k, v in times.items()},
               "ms_max": {k: round(max(v), 3) for k, v in times.items()},
               "conv_ms_per_launch": conv_layers(model, net, 2 * B * T, H, W, args.reps),
               "max_rel_frame_diff_from_calculate_lpips": diffs}
        print(json.dumps(res))


if __name__ == "__main__":
    main()
