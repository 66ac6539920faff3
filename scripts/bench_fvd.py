#!/usr/bin/env python
"""The FVD leg of vqgan_eval.py's video loop for one cfg-3 eval batch (8 clips x 17 x 256^2), seeded tokenizer and
seeded I3D weights (oracle/i3d_oracle.py weights with the BatchNorm statistics of tests/golden/fvd_i3d.pt).

    python scripts/bench_fvd.py [--rounds 5]

Arms, in alternating rounds, each step ending in a synchronise:
- (a) the script's way (vqgan_eval.py:114-148): the loader's normalised fp32 clip to the device, forward(log_image=True),
  the reconstruction to the host, the script's byte conversions, fvd.py's preprocess twice on the host (torch, default
  threads), the fp32 clips to the device, and I3D as torch ops on the GPU (cuDNN, TF32 allowed: torch's defaults);
- (b) consumers.eval_step_fvd from the loader's uint8 clip (host, pinned) copied to the device.
Reports ms per batch of each leg, the I3D device time of (b) (CUDA events, both calls), its algorithmic TFLOP/s from
the layer shapes, the MMA work omt_conv3d issues (tiles x tile size x K padded, per tf32 pass) against the algorithmic
work, and max |logit difference| of (a), (b) and strict fp32 cuDNN.  Prints ONE JSON line with the card's name, power
limit and max SM clock.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import omnitokenizer_b200 as ob  # noqa: E402
from omnitokenizer_b200 import consumers as C  # noqa: E402
from omnitokenizer_b200 import fvd  # noqa: E402
from omnitokenizer_b200 import layout as L  # noqa: E402
from oracle import i3d_oracle as io  # noqa: E402
from oracle import omni_oracle as oo  # noqa: E402
from oracle import weights as W  # noqa: E402
from scripts.bench_ingest import card  # noqa: E402

B, T, S = 8, 17, 256


def work(B, T):
    """(algorithmic FLOP, issued MMA FLOP of one tf32 pass) of I3D's convolutions on B clips of T frames at 224^2."""
    algo = issued = 0
    shape = (T, 224, 224)

    def conv(cin, cout, k, s, shape):
        nonlocal algo, issued
        _, o = fvd.same_geometry((k,) * 3, (s,) * 3, shape)
        M = B * o[0] * o[1] * o[2]
        K = L.round_up(k ** 3 * fvd.cpad(cin), 32)
        bn = 64 if cout <= 64 else 128
        algo += 2 * M * cout * cin * k ** 3
        issued += 2 * L.round_up(M, 128) * L.round_up(cout, bn) * K
        return o

    for name, kind, spec in fvd.ARCH:
        if kind == "unit":
            shape = conv(spec[0], spec[1], spec[2], spec[3], shape)
        elif kind == "pool":
            shape = fvd.same_geometry(spec[0], spec[1], shape)[1]
        else:
            cin, w = spec
            for b, (wi, k, src) in fvd.BRANCHES.items():
                conv(cin if src in ("x", "p") else w[fvd.BRANCHES[src][0]], w[wi], k, 1, shape)
    return algo, issued


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_fvd.py measures on a GPU"
    dev = torch.device("cuda:0")

    margs = ob.canonical_args()
    m = ob.OmniTokenizer_VQGAN(margs)
    m.load_state_dict(W.make_state_dict(oo.Config.from_args(margs), 0), strict=False)
    m.codebook._need_init = False
    m = m.to(dev).eval()
    golden = torch.load(os.path.join(ROOT, "tests", "golden", "fvd_i3d.pt"))
    sd = io.make_state_dict(golden["w_seed"])
    sd.update(golden["bn"])
    i3d = fvd.I3D(sd, dev)
    sd_dev = {k: v.to(dev) for k, v in sd.items()}

    u8 = torch.randint(0, 256, (B, T, S, S, 3), generator=torch.Generator().manual_seed(1), dtype=torch.uint8)
    u8_pin = u8.pin_memory()
    video = L.u8_normalize(u8, C.VIDEO_NORM)              # the loader's normalised clip, (B, 3, T, H, W) fp32, host

    def arm_a():
        t = [time.perf_counter()]
        with torch.no_grad():
            _, _, _, x_recons, _ = m(video.to(dev), log_image=True)
            torch.cuda.synchronize()
            t.append(time.perf_counter())
            real = ((video + 0.5) * 255).movedim(1, -1).byte().numpy()
            fake = (torch.clamp(x_recons.cpu() + 0.5, 0, 1) * 255).movedim(1, -1).byte().numpy()
            t.append(time.perf_counter())
            xr, xf = io.preprocess(real), io.preprocess(fake)
            t.append(time.perf_counter())
            xr, xf = xr.to(dev), xf.to(dev)
            torch.cuda.synchronize()
            t.append(time.perf_counter())
            lr, lf = io.forward(sd_dev, xr), io.forward(sd_dev, xf)
            torch.cuda.synchronize()
            t.append(time.perf_counter())
        legs = dict(zip(("forward", "d2h_bytes", "preprocess_x2", "h2d", "i3d_x2"), np.diff(t) * 1e3))
        return legs, lr, lf, (xr, xf)

    def arm_b():
        t0 = time.perf_counter()
        lr, lf, _ = C.eval_step_fvd(m, u8_pin.to(dev, non_blocking=True), i3d)
        torch.cuda.synchronize()
        return {"total": (time.perf_counter() - t0) * 1e3}, lr, lf

    for _ in range(3):                                     # warm-up: graphs captured, cuDNN algorithms picked
        arm_a(), arm_b()
    ra, rb = [], []
    for _ in range(args.rounds):
        ra.append(arm_a())
        rb.append(arm_b())
    legs_a = {k: float(np.median([r[0][k] for r in ra])) for k in ra[0][0]}
    total_a = float(np.median([sum(r[0].values()) for r in ra]))
    total_b = float(np.median([r[0]["total"] for r in rb]))

    # I3D device time of (b): both calls (real with the byte map, fake), CUDA events over 10 replays
    fake = m.forward_u8(u8_pin.to(dev), C.VIDEO_NORM, C.EVAL_U8)[0]
    frames = u8_pin.to(dev)
    a_ev, b_ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a_ev.record()
    for _ in range(10):
        i3d.logits(frames, real_norm=C.VIDEO_NORM)
        i3d.logits(fake)
    b_ev.record()
    torch.cuda.synchronize()
    i3d_ms = a_ev.elapsed_time(b_ev) / 10
    algo, issued = work(2 * B, T)

    # logits: (a), (b), strict fp32 cuDNN on (a)'s preprocessed clips
    _, la_r, la_f, (xr, xf) = ra[-1]
    _, lb_r, lb_f = rb[-1]
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    with torch.no_grad():
        ls_r, ls_f = io.forward(sd_dev, xr), io.forward(sd_dev, xf)
    torch.backends.cudnn.allow_tf32 = tf32
    la, lb, ls = torch.cat([la_r, la_f]), torch.cat([lb_r, lb_f]), torch.cat([ls_r, ls_f])
    d = lambda x, y: float((x - y).abs().max())
    out = {
        "metric": "fvd_leg_ms_per_batch", "workload": f"cfg3 eval batch: {B} real + {B} fake clips {T}x{S}x{S}",
        "a_script_ms": round(total_a, 2), "a_legs_ms": {k: round(v, 2) for k, v in legs_a.items()},
        "b_eval_step_fvd_ms": round(total_b, 2), "speedup": round(total_a / total_b, 2),
        "b_i3d_device_ms": round(i3d_ms, 3), "i3d_algorithmic_tflop": round(algo / 1e12, 3),
        "i3d_algorithmic_tflops_per_s": round(algo / (i3d_ms * 1e-3) / 1e12, 1),
        "issued_over_algorithmic_mma": round(issued / algo, 3),
        "max_abs_logit": round(float(ls.abs().max()), 4),
        "max_dlogit_a_b": d(la, lb), "max_dlogit_b_fp32": d(lb, ls), "max_dlogit_a_fp32": d(la, ls),
        "card": card(),
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
