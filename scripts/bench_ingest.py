#!/usr/bin/env python
"""Input side of the pipeline: uint8 frames into encode, with the loader's normalisation on the host or in the patch gather.

    python scripts/bench_ingest.py [--workloads cfg3,cfg2] [--steps 10] [--reps 20]

For each workload (bench.py's cfg3: 8 videos 17x256x256; cfg2: 64 images 256x256), on seeded uint8 frames:
- host: ms per batch of the reference loader's conversion -- cfg3: DecordVideoDataset.__getitem__ (OmniTokenizer/data.py:229-232:
  float, permute, VideoNorm, permute) per clip, cfg2: ToTensor + Normalize (data.py:88-97) per image -- then the collate
  (torch.stack), with 1 thread and with torch's default thread count;
- h2d: bytes and copy time (CUDA events) of the batch from pinned memory, fp32 against uint8;
- gather: device time (CUDA events, mean over --reps) of the first-frame + rest-frame patch gathers as encode launches them
  (row-scaled f16x3 planes), omt_patchify_ln against omt_patchify_ln_u8 (+ omt_u8_norm_select for VideoNorm);
- e2e: frames/s of two pipelines with bench.py's 3-stream overlap (H2D of step i+1 and D2H of step i-1 on their own
  streams): "u8" = pinned uint8 -> H2D -> encode_u8 -> decode_u8 -> D2H; "host_norm" = pinned uint8 -> host conversion
  (default threads) into pinned fp32 -> H2D -> encode -> decode_u8 -> D2H.
Prints ONE JSON line with the card's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {"cfg3": (8, 17, 256, 256, 3), "cfg2": (64, 256, 256, 3)}     # uint8, channels last (B, [T,] H, W, C)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clk = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:          # the measurement still stands; the card is then named by torch only
        return {"name": torch.cuda.get_device_name(), "power_limit": f"unknown ({e.__class__.__name__})"}


def host_convert(frames_u8, is_image, out=None):
    """The reference loader's per-sample conversion + collate; frames_u8 (B, [T,] H, W, 3) uint8 -> (B, 3, [T,] H, W) fp32."""
    from torchvision import transforms
    if is_image:
        tf = transforms.Compose([transforms.ToTensor(), transforms.Normalize((0.5, 0.5, 0.5), (1.0, 1.0, 1.0))])
        items = [tf(f.numpy()) for f in frames_u8]
    else:
        mean = torch.tensor([0.5, 0.5, 0.5]).view(1, 3, 1, 1)
        std = torch.tensor([1.0, 1.0, 1.0]).view(1, 3, 1, 1)
        items = []
        for f in frames_u8:
            vid = torch.from_numpy(f.numpy()).float().permute(0, 3, 1, 2)    # data.py:229-231
            if torch.max(vid) > 1 and mean.max() <= 1:                       # VideoNorm, video_utils.py:52-56
                vid.div_(255.0)
            items.append(vid.sub_(mean).div_(std).permute(1, 0, 2, 3))      # data.py:232
    return torch.stack(items, out=out)


def ev_ms(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def run(wl, args, dev):
    import omnitokenizer_b200 as ob
    from omnitokenizer_b200 import _cabi, consumers as C
    from omnitokenizer_b200 import layout as L
    from omnitokenizer_b200.engine import Planes

    shape = SHAPES[wl]
    is_image = len(shape) == 4
    B = shape[0]
    frames_per_step = B * (1 if is_image else shape[1])
    norm = C.IMAGE_NORM if is_image else C.VIDEO_NORM
    u8_host = torch.randint(0, 256, shape, generator=torch.Generator().manual_seed(5), dtype=torch.uint8).pin_memory()
    res = {"shape_u8": list(shape)}

    # ---- host conversion
    host = {}
    for label, threads in (("1_thread", 1), ("default_threads", torch.get_num_threads())):
        old = torch.get_num_threads()
        torch.set_num_threads(threads)
        host_convert(u8_host[:1], is_image)
        t0 = time.perf_counter()
        n = 3
        for _ in range(n):
            x = host_convert(u8_host, is_image)
        host[label] = {"threads": threads, "ms_per_batch": round((time.perf_counter() - t0) * 1e3 / n, 2)}
        torch.set_num_threads(old)
    res["host"] = host
    x_host = x.contiguous().pin_memory()
    # the uint8 path must hand the encoder the same fp32 values
    assert torch.equal(L.u8_normalize(u8_host.unsqueeze(1) if is_image else u8_host, norm).reshape(x_host.shape), x_host)

    # ---- H2D from pinned memory
    x_dev = torch.empty(x_host.shape, device=dev)
    u_dev = torch.empty(shape, device=dev, dtype=torch.uint8)
    res["h2d"] = {"fp32_bytes": x_host.numel() * 4, "u8_bytes": u8_host.numel(),
                  "fp32_ms": round(ev_ms(lambda: x_dev.copy_(x_host, non_blocking=True), args.reps), 3),
                  "u8_ms": round(ev_ms(lambda: u_dev.copy_(u8_host, non_blocking=True), args.reps), 3)}

    # ---- patch gathers (first + rest frames) into row-scaled planes
    m = ob.OmniTokenizer_VQGAN(ob.canonical_args())
    m.codebook._need_init = False
    m = m.to(dev).eval()
    eng = m.prepare().engine()
    T = 1 if is_image else shape[1]
    H = shape[-3]
    xv = x_dev.view(B, 3, T, H, H)
    uv = u_dev.view(B, T, H, H, 3)
    p, pt = eng.p, eng.pt
    kmax = 3 * pt * p * p
    rows = B * (T - 1) // pt * (H // p) ** 2 if T > 1 else B * (H // p) ** 2
    pl = Planes(dev, rows, kmax, row_scaled=True)
    lut = L.u8_norm_table(norm, 3).to(dev)
    sel = torch.empty(B, device=dev, dtype=torch.int32) if norm.max_test else None
    forms = [(1, eng.pe["first"])] + ([(0, eng.pe["rest"])] if T > 1 else [])

    def g32():
        for first, pe in forms:
            _cabi.call("omt_patchify_ln", xv, None, pl.hi, pl.lo, pl.rs, pe["ln1_g"], pe["ln1_b"], B, 3, T, H, H, p, pt, first, 1e-5)

    def g8():
        if sel is not None:
            _cabi.call("omt_u8_norm_select", uv, B, T * H * H * 3, sel)
        for first, pe in forms:
            _cabi.call("omt_patchify_ln_u8", uv, lut, sel, None, pl.hi, pl.lo, pl.rs, pe["ln1_g"], pe["ln1_b"], B, 3, T, H, H, p, pt,
                       first, 1e-5)

    x_dev.copy_(x_host)
    u_dev.copy_(u8_host)
    g32a, g8a, g32b, g8b = ev_ms(g32, args.reps), ev_ms(g8, args.reps), ev_ms(g32, args.reps), ev_ms(g8, args.reps)
    res["gather_us"] = {"patchify_ln_fp32": [round(g32a * 1e3, 1), round(g32b * 1e3, 1)],
                        "patchify_ln_u8": [round(g8a * 1e3, 1), round(g8b * 1e3, 1)], "note": "two alternating runs each"}
    del pl

    # ---- e2e, bench.py's 3-stream overlap
    main = torch.cuda.current_stream()
    s_in, s_out = torch.cuda.Stream(), torch.cuda.Stream()
    out_shape = (B, T, H, H, 3)
    oh = [torch.empty(out_shape, dtype=torch.uint8).pin_memory() for _ in range(2)]
    xpin = [torch.empty(x_host.shape).pin_memory() for _ in range(2)]

    def pipeline(nsteps, u8):
        src = [torch.empty(shape, device=dev, dtype=torch.uint8) if u8 else torch.empty(x_host.shape, device=dev) for _ in range(2)]
        ev_in, ev_used, ev_out = ([torch.cuda.Event() for _ in range(2)] for _ in range(3))
        keep = []
        for i in range(nsteps):
            sl = i & 1
            if not u8:
                if i >= 2:
                    ev_in[sl].synchronize()                      # the pinned buffer of step i-2 has been copied
                host_convert(u8_host, is_image, out=xpin[sl])
            with torch.cuda.stream(s_in):
                if i >= 2:
                    s_in.wait_event(ev_used[sl])
                src[sl].copy_(u8_host if u8 else xpin[sl], non_blocking=True)
                ev_in[sl].record(s_in)
            main.wait_event(ev_in[sl])
            if u8:
                codes = m.encode_u8(src[sl], is_image, norm=norm)
            else:
                codes = m.encode(src[sl], is_image)
            rec = m.decode_u8(codes, is_image)
            ev_used[sl].record(main)
            rec.record_stream(s_out)
            keep.append(rec)
            with torch.cuda.stream(s_out):
                s_out.wait_event(ev_used[sl])
                oh[sl].copy_(rec, non_blocking=True)
                ev_out[sl].record(s_out)
            if len(keep) > 3:
                keep.pop(0)
        for sl in range(2):
            main.wait_event(ev_out[sl])

    e2e = {}
    for rnd in range(2):                                         # alternate the two pipelines, twice
        for name, u8 in (("u8", True), ("host_norm", False)):
            pipeline(4, u8)
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            a.record(main)
            pipeline(args.steps, u8)
            b.record(main)
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            e2e.setdefault(name, []).append({"frames_per_s": round(frames_per_step * args.steps / (a.elapsed_time(b) / 1e3), 1),
                                             "wall_frames_per_s": round(frames_per_step * args.steps / wall, 1)})
    res["e2e"] = e2e
    # the two pipelines' codes agree on this batch
    c8 = m.encode_u8(u8_host.to(dev), is_image, norm=norm)
    c32 = m.encode(x_host.to(dev), is_image)
    res["codes_equal"] = bool(torch.equal(c8, c32))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg3,cfg2")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ingest.py measures on the GPU; there is no CPU mode"
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    out = {"card": card(), "math": os.environ.get("OMT_MATH", "f16x3"), "host_cpus": os.cpu_count(),
           "torch_threads": torch.get_num_threads()}
    for wl in [w for w in args.workloads.split(",") if w]:
        out[wl] = run(wl, args, dev)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
