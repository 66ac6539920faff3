"""Encode + decode throughput at every model width the kernels take, with the canonical 512 as the anchor, in one process:
   python scripts/bench_widths.py [--widths 256,512,768,1024] [--rounds R] [--steps S] [--batch B]

Workload: encode -> decode of B x 17 x 256^2 clips (default B = 8), the canonical flags with --embedding_dim C and
--heads C / 64 (so the window blocks keep 64-wide heads), seeded synthetic weights.  One model per width with two engines,
f16x3 and f16x1.  Every (width, mode) is warmed up (eager call, graph capture, replays); then R rounds run every
(width, mode) once each, the order rotated from round to round, each timed window S steps between CUDA events after an
untimed L2 flush.  Per (width, mode): median / min / max ms per step over the rounds, frames/s at the median, and the
algorithmic TFLOP/s: the multiply-adds the shapes imply (every nn.Linear, the attention products QK^T and PV, PEG, the
codebook distances; flops() below) over the median step time.  That is an end-to-end rate, not a kernel share of peak.
The card's name, power limit and max SM clock are read in the same call.  Prints ONE JSON line."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import omnitokenizer_b200 as ob  # noqa: E402
from omnitokenizer_b200.engine import Engine  # noqa: E402
from oracle import omni_oracle as oo  # noqa: E402
from oracle import weights as W  # noqa: E402
from scripts.bench_math import card  # noqa: E402

MODES = ("f16x3", "f16x1")


def flops(cfg: oo.Config, B: int, T: int, side: int) -> float:
    """Multiply-adds x 2 of one encode + decode of B x T x side^2 clips."""
    p, pt = cfg.patch_size, cfg.temporal_patch_size
    Tp, N = 1 + (T - 1) // pt, (side // p) ** 2
    M, C, A, inner, D = B * Tp * N, cfg.embedding_dim, cfg.heads * cfg.dim_head, cfg.ff_inner, cfg.dim_head
    k1, k2 = cfg.image_channels * p * p, cfg.image_channels * pt * p * p
    ff = 2 * M * C * 2 * inner + 2 * M * inner * C

    def t_layer(temporal):
        attn = 4 * D * cfg.heads * (B * N * Tp * Tp if temporal else B * Tp * N * N)
        return 2 * 27 * M * C + 2 * M * C * 3 * A + attn + 2 * M * A * C + ff

    def w_layer():
        ws = cfg.twod_window_size ** 2
        return 2 * M * C * 3 * C + 4 * ws * ws * (C // cfg.heads) * cfg.heads * (M // ws) + 2 * M * C * C + ff

    def tr(block, temporal):
        return sum(t_layer(temporal) if b == "t" else w_layer() for b in block)

    patches = 2 * B * N * C * k1 + 2 * B * (Tp - 1) * N * C * k2
    enc = patches + tr(cfg.enc_block, False) + tr("t" * cfg.temporal_depth, True)
    vq = 2 * M * C * cfg.codebook_dim + 2 * M * cfg.codebook_dim * cfg.n_codes
    dec = 2 * M * cfg.codebook_dim * C + tr("t" * cfg.temporal_depth, True) + tr(cfg.dec_block, False) + patches
    return float(enc + vq + dec)


def make_model(C, dev):
    argv = ["--embedding_dim", str(C), "--heads", str(C // 64)]
    args = ob.canonical_args(argv)
    cfg = oo.Config.from_args(args)
    m = ob.OmniTokenizer_VQGAN(args)
    res = m.load_state_dict(W.make_state_dict(cfg, 0), strict=False)
    assert not res.missing_keys and not res.unexpected_keys
    m.codebook._need_init = False
    return m.to(dev).eval(), cfg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--widths", default="256,512,768,1024")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--batch", type=int, default=8)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_widths.py measures on a GPU"
    dev = torch.device("cuda:0")
    widths = [int(w) for w in args.widths.split(",")]
    if 512 not in widths:
        widths.append(512)                       # the anchor always runs
    B, T, side = args.batch, 17, 256
    x = (torch.rand((B, 3, T, side, side), generator=torch.Generator().manual_seed(1234)) - 0.5).to(dev)
    runs = {}
    with torch.no_grad():
        for C in widths:
            m, cfg = make_model(C, dev)
            engines = {mode: Engine(m, dev, mode) for mode in MODES}
            for mode in MODES:
                m._engine = engines[mode]
                for _ in range(3):               # eager, capture, replay
                    m.decode(m.encode(x, False), False)
            runs[C] = (m, cfg, engines)
        torch.cuda.synchronize()
        flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)      # larger than the 50 MB L2
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        order = [(C, mode) for C in widths for mode in MODES]
        times = {k: [] for k in order}
        for r in range(args.rounds):
            k0 = r % len(order)
            for C, mode in order[k0:] + order[:k0]:
                m, _, engines = runs[C]
                m._engine = engines[mode]
                flush.zero_()
                torch.cuda.synchronize()
                start.record()
                for _ in range(args.steps):
                    m.decode(m.encode(x, False), False)
                end.record()
                torch.cuda.synchronize()
                times[(C, mode)].append(start.elapsed_time(end) / args.steps)
    frames = B * T
    results = []
    for C, mode in order:
        ts = sorted(times[(C, mode)])
        med = ts[len(ts) // 2]
        fl = flops(runs[C][1], B, T, side)
        results.append({"embedding_dim": C, "heads": C // 64, "math": mode, "ms_median": round(med, 3),
                        "ms_min": round(ts[0], 3), "ms_max": round(ts[-1], 3),
                        "frames_per_s_median": round(frames / (med * 1e-3), 1), "algorithmic_tflop_per_step": round(fl / 1e12, 3),
                        "algorithmic_tflops_median": round(fl / (med * 1e-3) / 1e12, 1)})
    anchor = {r["math"]: r["ms_median"] for r in results if r["embedding_dim"] == 512}
    for r in results:
        r["time_vs_512"] = round(r["ms_median"] / anchor[r["math"]], 3)
    print(json.dumps({"card": card(), "workload": f"encode+decode {B}x{T}x{side}^2", "rounds": args.rounds,
                      "steps_per_round": args.steps, "results": results}), flush=True)


if __name__ == "__main__":
    main()
