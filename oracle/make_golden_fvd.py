"""Generate tests/golden/fvd_i3d.pt from the UNMODIFIED reference FVD code (OmniTokenizer/fvd/pytorch_i3d.py and
fvd.py's preprocess / frechet_distance), loaded through oracle/ref_loader.py.

Weights: oracle.i3d_oracle.make_state_dict (torch.rand + exact arithmetic), with BatchNorm statistics calibrated on the
first clip so every unit's output is O(1); the statistics are stored in the fixture with a fingerprint of the weights.
Clips (uint8, seeded): 17 x 256^2 (downscale), 9 x 64^2 (upscale, the shortest clip the reference's AvgPool3d takes),
17 x 240 x 320 (UCF's size), 33 x 97 x 131 (odd sizes) and a constant clip (the padding decides the border).
When the real i3d_pretrained_400.pt is present, the oracle is also checked against the reference on it (printed only).

    python -m oracle.make_golden_fvd
"""
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402
from oracle import i3d_oracle as io  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "fvd_i3d.pt")
CLIPS = [("down_17x256", (17, 256, 256), 11), ("up_9x64", (9, 64, 64), 12), ("ucf_17x240x320", (17, 240, 320), 13),
         ("odd_33x97x131", (33, 97, 131), 14), ("const_9x80x96", (9, 80, 96), None)]
W_SEED = 5


def clip_bytes(shape, seed):
    if seed is None:
        return torch.full(shape + (3,), 200, dtype=torch.uint8)
    return torch.randint(0, 256, shape + (3,), generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)


def load_reference():
    ref_loader.load()                      # stubs + the OmniTokenizer package without its __init__
    sys.modules.setdefault("OmniTokenizer.modules.lpips",
                           types.SimpleNamespace(normalize_tensor=lambda x, eps=1e-10: x))
    if "sklearn" not in sys.modules:
        try:
            import sklearn.metrics.pairwise  # noqa: F401
        except ImportError:              # polynomial_mmd only; not used here
            for n in ("sklearn", "sklearn.metrics"):
                sys.modules[n] = types.ModuleType(n)
            sys.modules["sklearn.metrics.pairwise"] = types.SimpleNamespace(polynomial_kernel=None)
    import OmniTokenizer.fvd.pytorch_i3d as pi3d
    import OmniTokenizer.fvd.fvd as fvd
    return pi3d, fvd


def main():
    pi3d, fvd = load_reference()
    torch.manual_seed(0)
    sd = io.make_state_dict(W_SEED)
    first = clip_bytes(CLIPS[0][1], CLIPS[0][2])[None]
    io.calibrate_bn(sd, io.preprocess(first.numpy()))
    net = pi3d.InceptionI3d(400, in_channels=3).eval()
    missing, unexpected = net.load_state_dict(sd, strict=True)
    out = {"w_seed": W_SEED, "fingerprint": io.conv_fingerprint(sd), "bn": io.bn_stats(sd), "clips": {}}
    worst = 0.0
    for name, shape, seed in CLIPS:
        u8 = clip_bytes(shape, seed)[None]
        with torch.no_grad():
            x = fvd.preprocess(u8.numpy(), fvd.TARGET_RESOLUTION)
            ref = net(x)
            eps = {}
            ora = io.forward(sd, io.preprocess(u8.numpy()), eps)
        rel = float((ora - ref).abs().max() / ref.abs().max())
        worst = max(worst, rel)
        print(f"{name}: logits max|ref| {float(ref.abs().max()):.3f}, oracle rel diff {rel:.2e}")
        g = torch.Generator().manual_seed(seed or 99)
        pi = torch.randint(0, x.numel(), (512,), generator=g)
        entry = {"shape": shape, "seed": seed, "logits": ref[0].clone(), "pre_idx": pi, "pre_val": x.flatten()[pi].clone()}
        if name == CLIPS[0][0]:
            entry["endpoints"] = {k: io.endpoint_summary(v, 1000 + i) for i, (k, v) in enumerate(eps.items())}
        out["clips"][name] = entry
    g = torch.Generator().manual_seed(21)
    a, b = torch.rand(12, 6, generator=g), torch.rand(12, 6, generator=g) * 1.5 + 0.25
    out["fd"] = {"x1": a, "x2": b, "value": fvd.frechet_distance(a, b)}
    print(f"frechet_distance {float(out['fd']['value']):.6f}, oracle {float(io.frechet_distance(a, b)):.6f}")

    real = os.path.join(ref_loader.REF_ROOT, "OmniTokenizer", "fvd", "i3d_pretrained_400.pt")
    if os.path.exists(real):
        rsd = torch.load(real, map_location="cpu")
        rnet = pi3d.InceptionI3d(400, in_channels=3).eval()
        rnet.load_state_dict(rsd)
        u8 = clip_bytes((17, 256, 256), 31)[None]
        with torch.no_grad():
            ref = rnet(fvd.preprocess(u8.numpy(), fvd.TARGET_RESOLUTION))
            ora = io.forward({k: v.float() for k, v in rsd.items()}, io.preprocess(u8.numpy()))
        print(f"real checkpoint ({len(rsd)} tensors): max|ref| {float(ref.abs().max()):.3f}, "
              f"oracle max|diff| {float((ora - ref).abs().max()):.2e}")
    torch.save(out, OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1e6:.2f} MB); worst oracle rel diff {worst:.2e}")


if __name__ == "__main__":
    main()
