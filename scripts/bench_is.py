"""The video-metric suite's Inception Score on one Latte-sized sample batch: 16 clips of 16 fp32 frames, 256 x 256, in
[0, 1] on the device.  iscore.calculate_is against the suite's way (calculate_is.py: per clip, nn.Upsample on the
device, torchvision's Inception3 on cuDNN fp32 with cudnn.allow_tf32 on (torch's default) and off, F.softmax to numpy,
then the scipy.stats.entropy loop on the host), in alternating rounds.  Both run the fixture's seeded weights
(tests/golden/is_inception.pt).  Reports frames/s and whole-call ms (median over rounds, host clock around calls that
end on the host), algorithmic TFLOP/s (from the layer shapes), and the max |probability| and IS differences against
each arm; one JSON line with the card, its power limit and max SM clock.

    python scripts/bench_is.py [--rounds 5]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from omnitokenizer_b200 import iscore  # noqa: E402
from oracle import is_oracle as io  # noqa: E402
from scripts.bench_fid import flop_per_image  # noqa: E402
from scripts.bench_ingest import card  # noqa: E402

B, T, S = 16, 16, 256


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_is.py measures on a GPU"
    import torchvision
    from scipy.stats import entropy
    dev = torch.device("cuda:0")
    golden = torch.load(os.path.join(ROOT, "tests", "golden", "is_inception.pt"), weights_only=False)
    sd = io.fixture_state_dict(golden)
    model = iscore.ISInception(sd, dev)
    tv = torchvision.models.Inception3(transform_input=False, aux_logits=True, init_weights=False)
    tv.load_state_dict(sd, strict=True)
    tv = tv.to(dev).eval()
    up = torch.nn.Upsample(size=(299, 299), mode="bilinear").to(dev)
    videos = io.frames((B * T, S, S), 5).view(B, T, 3, S, S).to(dev)
    last = {}

    def ours():
        last["omt_is"] = None
        return iscore.calculate_is(videos, dev, 1, model=model)

    def suite(name):
        preds = np.zeros((B * T, 1000))
        with torch.no_grad():
            for i, batch in enumerate(videos):
                preds[i * T:(i + 1) * T] = F.softmax(tv(up(batch)), dim=1).cpu().numpy()
        last[name] = preds
        py = np.mean(preds, axis=0)
        s = np.exp(np.mean([entropy(preds[i], py) for i in range(preds.shape[0])]))
        return np.mean([s]), np.std([s])

    arms = {"omt_is": (ours, True), "suite_cudnn_tf32": (lambda: suite("suite_cudnn_tf32"), True),
            "suite_cudnn_fp32": (lambda: suite("suite_cudnn_fp32"), False)}

    def run(fn, tf32):
        torch.backends.cudnn.allow_tf32 = tf32
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()                                    # ends on the host: the scores are numpy values
        return (time.perf_counter() - t0) * 1e3, r

    for _ in range(2):                              # warm-up: workspaces and graphs, cuDNN algorithms
        for fn, tf32 in arms.values():
            run(fn, tf32)
    ms = {k: [] for k in arms}
    res = {}
    for _ in range(args.rounds):
        for k, (fn, tf32) in arms.items():
            t, res[k] = run(fn, tf32)
            ms[k].append(t)
    torch.backends.cudnn.allow_tf32 = True
    probs = model.probabilities(videos.view(B * T, 3, S, S)).double().cpu().numpy()
    flop = flop_per_image() + 2 * iscore.FEATURES * iscore.NUM_CLASSES
    med = {k: float(np.median(v)) for k, v in ms.items()}
    N = B * T
    out = {
        "metric": "inception_score_frames_per_s", "workload": f"calculate_is on {B} clips of {T} fp32 frames {S}x{S}",
        "frames_per_s": {k: round(N / (v * 1e-3), 1) for k, v in med.items()},
        "ms_per_call": {k: round(v, 2) for k, v in med.items()},
        "ms_per_call_range": {k: [round(min(v), 2), round(max(v), 2)] for k, v in ms.items()},
        "speedup_vs_suite_tf32": round(med["suite_cudnn_tf32"] / med["omt_is"], 2),
        "speedup_vs_suite_fp32": round(med["suite_cudnn_fp32"] / med["omt_is"], 2),
        "gflop_per_frame": round(flop / 1e9, 2),
        "algorithmic_tflops_per_s": {k: round(N * flop / (v * 1e-3) / 1e12, 1) for k, v in med.items()},
        "is": {k: [float(v[0]), float(v[1])] for k, v in res.items()},
        "max_dprob_vs_suite_tf32": float(np.abs(probs - last["suite_cudnn_tf32"]).max()),
        "max_dprob_vs_suite_fp32": float(np.abs(probs - last["suite_cudnn_fp32"]).max()),
        "is_rel_diff_vs_suite_tf32": abs(float(res["omt_is"][0]) / float(res["suite_cudnn_tf32"][0]) - 1),
        "is_rel_diff_vs_suite_fp32": abs(float(res["omt_is"][0]) / float(res["suite_cudnn_fp32"][0]) - 1),
        "rounds": args.rounds,
        "card": card(),
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
