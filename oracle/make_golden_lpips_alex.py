"""Generate tests/golden/lpips_alex.pt from the UNMODIFIED evaluation/common_metrics_on_video_quality/calculate_lpips.py,
loaded by file path.

The suite builds `loss_fn = lpips.LPIPS(net='alex', spatial=True)` when it is imported.  The lpips package is not in the
reference tree, so before the import a stub `lpips` module goes into sys.modules: its LPIPS(net, spatial) asserts
('alex', True) and returns oracle.lpips_alex_oracle.AlexLPIPSOracle carrying the seeded weights of its
make_state_dict, which records each frame's value as the suite takes it.  The maker then calls the suite's
calculate_lpips(v1, v2, torch.device('cpu')).

What this pins: the suite's loop, trans (grey repeated to 3 channels, x * 2 - 1), the per-frame .mean() and the result
dict, by running the suite's own file.  What it does not: the lpips package's own arithmetic (ScalingLayer,
normalize_tensor, the lin layers, the upsample and the tap sum), which only the restatement in lpips_alex_oracle.py
states; the trunk is the installed torchvision's alexnet().features.  The fixture holds a fingerprint of the weights,
not the weights; the inputs are regenerated from their specs (lpips_alex_oracle.videos).

    python -m oracle.make_golden_lpips_alex
"""
import importlib.util
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import lpips_alex_oracle as ao  # noqa: E402
from oracle.ref_loader import REF_ROOT  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "lpips_alex.pt")
SUITE = os.path.join(REF_ROOT, "evaluation", "common_metrics_on_video_quality", "calculate_lpips.py")
W_SEED = 11
# name -> (B, T, C, H, W, kind, seed)
CASES = {
    "demo_zeros_ones_64": (2, 3, 3, 64, 64, "zeros_ones", 0),
    "bytes_64": (2, 2, 3, 64, 64, "bytes", 1),
    "bytes_256": (1, 2, 3, 256, 256, "bytes", 2),
    "bytes_67x93": (2, 2, 3, 67, 93, "bytes", 3),
    "min_31": (2, 2, 3, 31, 31, "bytes", 4),
    "min_31x45": (1, 3, 3, 31, 45, "bytes", 5),
    "border_64": (1, 2, 3, 64, 64, "border", 9),
    "float_48x40": (2, 2, 3, 48, 40, "float", 6),
    "grey_64": (2, 2, 1, 64, 64, "float", 7),
    "same_64": (1, 2, 3, 64, 64, "same", 8),
}
MAPS_CASE = "min_31x45"             # its five tap maps and the spatial map of its first frame are stored


def load_suite(net):
    """calculate_lpips.py, imported with a stub lpips package whose LPIPS is `net`."""
    def LPIPS(**kw):
        assert kw == {"net": "alex", "spatial": True}, kw
        return net

    sys.modules["lpips"] = types.SimpleNamespace(LPIPS=LPIPS)
    spec = importlib.util.spec_from_file_location("omt_ref_calculate_lpips", SUITE)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    sd = ao.make_state_dict(W_SEED)
    net = ao.AlexLPIPSOracle(sd).eval()
    suite = load_suite(net)
    out = {"w_seed": W_SEED, "fingerprint": ao.fingerprint(sd), "maps_case": MAPS_CASE, "cases": {}}
    for name, spec in CASES.items():
        v1, v2 = ao.videos(spec)
        net.record = []
        net.maps = [] if name == MAPS_CASE else None
        with torch.no_grad():
            r = suite.calculate_lpips(v1, v2, torch.device("cpu"))
        per = torch.tensor(net.record, dtype=torch.float64).view(spec[0], spec[1])
        e = {"spec": spec, "per_frame": per, "value": {t: float(v) for t, v in r["value"].items()},
             "value_std": {t: float(v) for t, v in r["value_std"].items()},
             "video_setting": tuple(r["video_setting"]), "video_setting_name": r["video_setting_name"]}
        if net.maps is not None:
            taps, val = net.maps[0]
            e["tap_maps"] = [t[0, 0].clone() for t in taps]
            e["map"] = val[0, 0].clone()
        out["cases"][name] = e
        print(f"{name}: per-frame {per.flatten().tolist()}")
    torch.save(out, OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1e3:.1f} kB)")


if __name__ == "__main__":
    main()
