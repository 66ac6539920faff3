"""Device time per kernel of one warmed bench step, from torch.profiler (CUDA activities):
   python scripts/kernel_breakdown.py [--math f16x3|f16x1|3xtf32|fp32] [--workload cfg3|cfg2|cfg4|cfg5] [--top N]

CUDA graphs are turned off (OMT_CUDA_GRAPH=0) so that every launch is its own event.  Kernels are grouped by name with
the template arguments kept (they tell the GEMM instantiations apart) and the parameter list dropped; each line gives
the launches, the device time, and the share of the step's summed device time.  For the f16x3 wgmma GEMM the script also
records the shape of every omt_linear_h call and prints the achieved f16 tensor rate, 3 x 2MNK (three f16 products per
fp32-grade product, launched N; 1 x 2MNK for the single-product f16x1 GEMM) over device time, next to the H100 SXM
data-sheet dense f16 figure of 989 TFLOP/s."""
import argparse
import collections
import os
import sys

os.environ["OMT_CUDA_GRAPH"] = "0"
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from omnitokenizer_b200 import _cabi  # noqa: E402

F16_DATASHEET_TFLOPS = 989.0


def kernel_name(name):
    """'void ns::k<a, b>(args...)' -> 'ns::k<a, b>'"""
    if name.startswith("void "):
        name = name[5:]
    depth = 0
    for i, ch in enumerate(name):
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            return name[:i]
    return name


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--math", default="f16x3")
    ap.add_argument("--workload", default="cfg3", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--top", type=int, default=25)
    args = ap.parse_args()
    os.environ["OMT_MATH"] = args.math
    assert torch.cuda.is_available(), "kernel_breakdown.py measures on a GPU"
    dev = torch.device("cuda:0")
    wl = bench.WORKLOADS[args.workload]
    shape = wl["shape"]
    is_image = len(shape) == 4
    vae = bool(wl.get("vae"))
    x = (torch.rand(shape, generator=torch.Generator().manual_seed(1234)) - 0.5).to(dev)
    m = bench.make_model(dev, vae)
    m.prepare()

    def step():
        z = m.encode(x, is_image)
        if vae and not is_image:
            z = z.permute(0, 2, 3, 4, 1)
        return m.decode(z, is_image)

    for _ in range(3):
        step()
    torch.cuda.synchronize()

    shapes = []                          # (M, N, K) of every omt_linear_h call of the profiled step, in launch order
    linear_h = _cabi.linear_h

    def recording_linear_h(*a, **kw):
        if kw["M"] > 0:                  # M == 0 launches nothing
            shapes.append((kw["M"], kw["N"], kw["K"]))
        return linear_h(*a, **kw)

    _cabi.linear_h = recording_linear_h
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        start.record()
        step()
        end.record()
        torch.cuda.synchronize()
    _cabi.linear_h = linear_h

    kernels = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA),
                     key=lambda e: e.time_range.start)
    total_us = sum(e.time_range.elapsed_us() for e in kernels)
    by_name = collections.defaultdict(lambda: [0, 0.0, 0.0])     # launches, us, f16 tensor flops
    gemms = [e for e in kernels if "gemm_wgmma_kernel<false" in e.name]
    rates = len(gemms) == len(shapes) and len(shapes) > 0
    for e in kernels:
        r = by_name[kernel_name(e.name)]
        r[0] += 1
        r[1] += e.time_range.elapsed_us()
    if rates:
        for e, (M, N, K) in zip(gemms, shapes):
            by_name[kernel_name(e.name)][2] += (1 if args.math == "f16x1" else 3) * 2.0 * M * N * K
    print(f"device: {torch.cuda.get_device_name(dev)}   workload {args.workload}   math {args.math}")
    print(f"step (CUDA events, profiler on): {start.elapsed_time(end):.2f} ms   summed kernel time: {total_us / 1e3:.2f} ms"
          f"   launches: {len(kernels)}")
    if not rates:
        print(f"(no f16 rates: {len(gemms)} f16 wgmma GEMM kernels, {len(shapes)} omt_linear_h calls)")
    print(f"{'ms':>9} {'share':>6} {'launches':>8} {'f16 TFLOP/s':>12}  kernel")
    for name, (n, us, fl) in sorted(by_name.items(), key=lambda kv: -kv[1][1])[:args.top]:
        rate = f"{fl / (us * 1e-6) / 1e12:7.1f} ({fl / (us * 1e-6) / 1e12 / F16_DATASHEET_TFLOPS:4.0%})" if fl else ""
        print(f"{us / 1e3:9.3f} {us / total_us:6.1%} {n:8d} {rate:>12}  {name}")
    if rates:
        print(f"f16 TFLOP/s: {1 if args.math == 'f16x1' else 3} x 2MNK over device time; (%) of the {F16_DATASHEET_TFLOPS:.0f} TFLOP/s H100 SXM data-sheet "
              f"dense f16 rate")


if __name__ == "__main__":
    main()
