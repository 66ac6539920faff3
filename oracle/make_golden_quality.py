"""Generate tests/golden/quality.pt from the UNMODIFIED reference metric code, loaded by file path:
evaluation/common_metrics_on_video_quality/calculate_psnr.py and calculate_ssim.py (numpy / cv2), and
OmniTokenizer/modules/lpips.py's LPIPS.

lpips.py builds its trunk with torchvision's models.vgg16(pretrained=True) and fetches its lin layers through
get_ckpt_path / load_from_pretrained.  Both are replaced, before LPIPS is built, by checked stubs: the module's `models`
is a namespace whose vgg16 asserts pretrained=True and returns an untrained torchvision vgg16 carrying the seeded
weights of oracle.quality_oracle.make_state_dict, and load_from_pretrained asserts it was asked for "vgg_lpips" and
loads the seeded lin weights, so nothing is downloaded.  The fixture stores a fingerprint of the weights, not the weights.

The suite's functions get the frames as float64 tensors holding the fp32 values byte / 255: its PSNR then runs in
float64 (on float32 input numpy would keep float32), as the device kernel does.
Cases (uint8 pairs regenerated from their spec by quality_oracle.frame_pair): noisy pairs at 256^2, 64^2 and 67 x 93,
the minimum sizes (11 x 11 for SSIM, 16 x 16 for LPIPS), an identical pair, a constant pair, and pairs differing in one
and in two bytes by 1 at 256^2 (mse 7.8e-11, under the PSNR rule's 1e-10, and 1.6e-10, over it).

    python -m oracle.make_golden_quality
"""
import importlib.util
import os
import sys
import types

import cv2
import numpy as np
import torch
import torchvision

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import quality_oracle as qo  # noqa: E402
from oracle.ref_loader import REF_ROOT  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "quality.pt")
METRICS = os.path.join(REF_ROOT, "evaluation", "common_metrics_on_video_quality")
LPIPS_SRC = os.path.join(REF_ROOT, "OmniTokenizer", "modules", "lpips.py")
W_SEED = 5
# name -> (H, W, kind, seed); lpips: whether the case is large enough for LPIPS
CASES = {
    "noise_256": ((256, 256, "noise", 1), True),
    "noise_64": ((64, 64, "noise", 2), True),
    "noise_67x93": ((67, 93, "noise", 3), True),
    "min_ssim_11": ((11, 11, "noise", 4), False),
    "min_lpips_16": ((16, 16, "noise", 5), True),
    "same_64": ((64, 64, "same", 6), True),
    "const_32": ((32, 32, "const", 7), True),
    "one_byte_256": ((256, 256, "one", 8), False),
    "two_bytes_256": ((256, 256, "two", 9), False),
}


def load_module(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def build_reference_lpips(lp, sd):
    """lpips.py's LPIPS() with sd as the weights its vgg16(pretrained=True) and load_from_pretrained would fetch."""
    def vgg16(pretrained=False, **kw):
        assert pretrained is True, "lpips.py asks for the pretrained trunk"
        m = torchvision.models.vgg16(weights=None)
        feats = {}
        for s, convs in enumerate(qo.VGG_SLICES, 1):
            for idx, _, _ in convs:
                feats[f"features.{idx}.weight"] = sd[f"net.slice{s}.{idx}.weight"]
                feats[f"features.{idx}.bias"] = sd[f"net.slice{s}.{idx}.bias"]
        missing, _ = m.load_state_dict(feats, strict=False)
        assert all(k.startswith("classifier.") for k in missing), missing
        return m

    def load_from_pretrained(self, name="vgg_lpips"):
        assert name == "vgg_lpips", name
        lin = {k: v.clone() for k, v in sd.items() if k.startswith("lin")}
        missing, unexpected = self.load_state_dict(lin, strict=False)
        assert not unexpected and all(not k.startswith("lin") for k in missing), (missing, unexpected)

    lp.models = types.SimpleNamespace(vgg16=vgg16)
    lp.LPIPS.load_from_pretrained = load_from_pretrained
    return lp.LPIPS().eval()


def main():
    psnr_mod = load_module("calculate_psnr", os.path.join(METRICS, "calculate_psnr.py"))
    ssim_mod = load_module("calculate_ssim", os.path.join(METRICS, "calculate_ssim.py"))
    lp = load_module("omt_ref_lpips", LPIPS_SRC)
    sd = qo.make_state_dict(W_SEED)
    net = build_reference_lpips(lp, sd)
    taps = torch.from_numpy(cv2.getGaussianKernel(11, 1.5).ravel().copy())
    out = {"w_seed": W_SEED, "fingerprint": qo.fingerprint(sd), "taps": taps, "cases": {}}
    worst = {"psnr": 0.0, "ssim": 0.0, "lpips": 0.0}
    for name, (spec, with_lpips) in CASES.items():
        a, b = qo.frame_pair(spec)
        a01, b01 = qo.to01(a)[None, None], qo.to01(b)[None, None]             # (1, 1, 3, H, W)
        p = psnr_mod.calculate_psnr(a01.double(), b01.double())["value"][0]
        s = ssim_mod.calculate_ssim(a01.double(), b01.double())["value"][0]
        e = {"spec": spec, "psnr": float(p), "ssim": float(s), "lpips": None}
        an, bn = a01[0, 0].double().numpy(), b01[0, 0].double().numpy()
        worst["psnr"] = max(worst["psnr"], abs(qo.psnr(an, bn) - p))
        worst["ssim"] = max(worst["ssim"], abs(qo.ssim(an, bn, taps.numpy()) - s))
        if with_lpips:
            with torch.no_grad():
                # calculate_lpips.trans (x * 2 - 1), then the tokenizer's LPIPS forward
                ref = net(a01[0] * 2 - 1, b01[0] * 2 - 1).flatten()
                per_tap, feats = [], []
                ora = qo.lpips(sd, a01[0], b01[0], per_tap=per_tap, features=feats)
            e["lpips"] = float(ref[0])
            e["lpips_taps"] = torch.stack([t[0] for t in per_tap])
            worst["lpips"] = max(worst["lpips"], abs(float(ora[0]) - float(ref[0])) / max(abs(float(ref[0])), 1e-30))
            if name == "noise_256":
                g = torch.Generator().manual_seed(77)
                ends = []
                for k, (fa, fb) in enumerate(feats):
                    rms = float(fa.pow(2).mean().sqrt())
                    print(f"  tap {k} ({tuple(fa.shape[1:])}): rms {rms:.3f}, max {float(fa.abs().max()):.3f}")
                    idx = torch.randint(0, fa.numel(), (64,), generator=g)
                    ends.append({"idx": idx, "a": fa.flatten()[idx].clone(), "b": fb.flatten()[idx].clone()})
                e["endpoints"] = ends
        out["cases"][name] = e
        print(f"{name}: psnr {p:.12g}  ssim {s:.12g}  lpips {e['lpips']}")
    torch.save(out, OUT)
    print(f"oracle vs reference: psnr {worst['psnr']:.2e} abs, ssim {worst['ssim']:.2e} abs, "
          f"lpips {worst['lpips']:.2e} rel")
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1e6:.3f} MB)")


if __name__ == "__main__":
    main()
