"""f16x1 (throughput mode) against f16x3 (the default) on the bench.py workloads, in one process:
   python scripts/bench_math.py [--workloads cfg3,cfg2,cfg4,cfg5] [--rounds R] [--steps S]

One model per workload (bench.make_model, bench.py's shapes and input seed) with two engines on it, one per math mode.
Every shape is warmed up on both engines (eager call, graph capture, replays).  Then R rounds alternate the two modes,
rotating which one starts a round; each timed window is S encode -> decode steps between CUDA events, after an untimed
L2 flush and ending in a device synchronise.  Per mode: median, min and max over the rounds, in ms per step and frames/s.

Accuracy on the same inputs, f16x1 against f16x3: code flips, max |dpx| of decoding f16x3's codes with each mode
(decoder alone) and of each mode's own round trip, or for VAE workloads the max |dz| of the latents drawn with the same
noise.  The card's name, power limit and max SM clock are read in the same call.  Prints ONE JSON line.

bench.py cannot run f16x1: its roofline table maps the three fp32-grade modes only (scripts/README.md)."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from omnitokenizer_b200.engine import Engine  # noqa: E402

MODES = ("f16x3", "f16x1")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        name, power, clk = [s.strip() for s in out.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:          # the measurement still stands; the card is then named by torch only
        return {"name": torch.cuda.get_device_name(), "power_limit": f"unknown ({e.__class__.__name__})"}


def run_workload(wl_name, dev, rounds, steps):
    wl = bench.WORKLOADS[wl_name]
    shape, vae = wl["shape"], bool(wl.get("vae"))
    is_image = len(shape) == 4
    frames = shape[0] * (1 if is_image else shape[2])
    x = (torch.rand(shape, generator=torch.Generator().manual_seed(1234)) - 0.5).to(dev)
    m = bench.make_model(dev, vae)
    m.prepare()
    engines = {mode: Engine(m, dev, mode) for mode in MODES}

    def use(mode):              # the module API runs on whichever engine it holds; both pack the same weights
        m._engine = engines[mode]

    def encode():
        if vae:
            torch.manual_seed(7)                 # the same posterior noise draw for both modes
        return m.encode(x, is_image)

    def decode(z):
        return m.decode(z.permute(0, 2, 3, 4, 1) if vae and not is_image else z, is_image)

    out = {}
    for mode in MODES:
        use(mode)
        for _ in range(3):                       # eager, capture, replay
            z = encode()
            rec = decode(z)
        torch.cuda.synchronize()
        out[mode] = (z.clone(), rec.clone())
    acc = {}
    (z3, r3), (z1, r1) = out["f16x3"], out["f16x1"]
    if vae:
        acc["max_abs_dz"] = float((z1 - z3).abs().max())
    else:
        acc["code_flips"] = int((z1 != z3).sum())
        acc["codes"] = z3.numel()
        use("f16x1")
        acc["max_abs_dpx_decoder"] = float((decode(z3) - r3).abs().max())
    acc["max_abs_dpx_round_trip"] = float((r1 - r3).abs().max())

    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)      # larger than the 50 MB L2
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = {mode: [] for mode in MODES}
    for r in range(rounds):
        for mode in (MODES if r % 2 == 0 else MODES[::-1]):
            use(mode)
            flush.zero_()
            torch.cuda.synchronize()
            start.record()
            for _ in range(steps):
                decode(encode())
            end.record()
            torch.cuda.synchronize()
            times[mode].append(start.elapsed_time(end) / steps)
    res = {"workload": wl_name, "desc": wl["desc"], "rounds": rounds, "steps_per_round": steps, "accuracy": acc}
    for mode in MODES:
        ts = sorted(times[mode])
        med = ts[len(ts) // 2]
        res[mode] = {"ms_median": round(med, 3), "ms_min": round(ts[0], 3), "ms_max": round(ts[-1], 3),
                     "frames_per_s_median": round(frames / (med * 1e-3), 1)}
    res["speedup_median"] = round(res["f16x3"]["ms_median"] / res["f16x1"]["ms_median"], 3)
    del engines, m
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg3,cfg2,cfg4,cfg5")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_math.py measures on a GPU"
    dev = torch.device("cuda:0")
    out = {"card": card(), "results": []}
    with torch.no_grad():
        for wl in args.workloads.split(","):
            out["results"].append(run_workload(wl, dev, args.rounds, args.steps))
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
