"""Generate tests/golden/fid_inception.pt from the UNMODIFIED reference FID code
(evaluation/pytorch-fid/src/pytorch_fid/inception.py and fid_score.calculate_frechet_distance), loaded by file path.

Weights: oracle.fid_oracle.make_state_dict (torch.rand + exact arithmetic), with BatchNorm statistics calibrated on the
five seeded random images so every unit's output is O(1); the statistics are stored in the fixture with a fingerprint
of the weights.  fid_score.py calls scipy.linalg.sqrtm(..., disp=False), an argument scipy 1.16 removed; on such a
scipy the module's `linalg` is a shim that takes it (scipy_linalg_with_disp).  fid_inception_v3() fetches its weights with load_state_dict_from_url(FID_WEIGHTS_URL): that module attribute
is replaced, before InceptionV3 is built, by a function that checks it was asked for that URL and returns the seeded
state dict, so nothing is downloaded.
Images (uint8, seeded): 256^2 (upscale), 128^2, 299^2 (identity size), 320 x 480 (downscale), 97 x 131 (odd sizes) and
a constant image.  When the real pt_inception-2015-12-05-6726825d.pth is in the torch hub cache, the oracle is also
checked against the reference on it (printed only).

    python -m oracle.make_golden_fid
"""
import importlib.util
import inspect
import os
import sys
import types

import numpy as np
import scipy.linalg
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import fid_oracle as fo  # noqa: E402
from oracle.ref_loader import REF_ROOT  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "fid_inception.pt")
FID_SRC = os.path.join(REF_ROOT, "evaluation", "pytorch-fid", "src", "pytorch_fid")
IMAGES = [("up_256", (256, 256), 11), ("up_128", (128, 128), 12), ("same_299", (299, 299), 13),
          ("down_320x480", (320, 480), 14), ("odd_97x131", (97, 131), 15), ("const_64x80", (64, 80), None)]
W_SEED = 7
WEIGHT_FILE = "pt_inception-2015-12-05-6726825d.pth"


def load_module(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def scipy_linalg_with_disp():
    """scipy.linalg whose sqrtm takes fid_score.py's `disp` argument: scipy 1.16 removed it.  disp=False returns
    (root, the Frobenius error estimate), as earlier scipy did."""
    if "disp" in inspect.signature(scipy.linalg.sqrtm).parameters:
        return scipy.linalg

    def sqrtm(a, disp=True):
        r = scipy.linalg.sqrtm(a)
        return r if disp else (r, np.linalg.norm(r.dot(r) - a, "fro") / np.linalg.norm(a, "fro"))

    return types.SimpleNamespace(sqrtm=sqrtm)


def build_reference(inception, sd):
    """InceptionV3([3]) (the 2048-wide pool3 features) with sd as the weights fid_inception_v3 fetches."""
    def fake_load(url, *a, **k):
        assert url == inception.FID_WEIGHTS_URL, url
        return {k_: v.clone() for k_, v in sd.items()}

    inception.load_state_dict_from_url = fake_load
    return inception.InceptionV3([inception.InceptionV3.BLOCK_INDEX_BY_DIM[2048]]).eval()


def main():
    inception = load_module("inception", os.path.join(FID_SRC, "inception.py"))   # fid_score.py: `from inception import`
    fid_score = load_module("pytorch_fid_score", os.path.join(FID_SRC, "fid_score.py"))
    fid_score.linalg = scipy_linalg_with_disp()
    torch.manual_seed(0)
    sd = fo.make_state_dict(W_SEED)
    cal = torch.cat([fo.preprocess(fo.image_bytes(shape, seed)[None]) for _, shape, seed in IMAGES if seed is not None])
    fo.calibrate_bn(sd, cal)
    net = build_reference(inception, sd)
    out = {"w_seed": W_SEED, "fingerprint": fo.conv_fingerprint(sd), "bn": fo.bn_stats(sd), "images": {}}
    worst = 0.0
    for name, shape, seed in IMAGES:
        u8 = fo.image_bytes(shape, seed)[None]
        x01 = u8.permute(0, 3, 1, 2).contiguous().float().div(255)        # fid_score.py:146 ToTensor
        with torch.no_grad():
            ref = net(x01)[0].squeeze(3).squeeze(2)                       # fid_score.py:163-170
            eps = {}
            ora = fo.forward(sd, fo.preprocess(u8), eps)
            # the reference's own preprocess (inception.py:147-151), for the sampled values
            pre = 2 * torch.nn.functional.interpolate(x01, size=(299, 299), mode="bilinear", align_corners=False) - 1
        rel = float((ora - ref).abs().max() / ref.abs().max())
        worst = max(worst, rel)
        print(f"{name}: features max|ref| {float(ref.abs().max()):.3f}, oracle rel diff {rel:.2e}")
        g = torch.Generator().manual_seed(seed or 99)
        pi = torch.randint(0, pre.numel(), (512,), generator=g)
        entry = {"shape": shape, "seed": seed, "features": ref[0].clone(), "pre_idx": pi, "pre_val": pre.flatten()[pi].clone()}
        if name == IMAGES[0][0]:
            entry["endpoints"] = {k: fo.endpoint_summary(v, 1000 + i) for i, (k, v) in enumerate(eps.items())}
        out["images"][name] = entry
    g = torch.Generator().manual_seed(21)
    a = torch.rand(40, 8, generator=g, dtype=torch.float64)
    b = torch.rand(40, 8, generator=g, dtype=torch.float64) * 1.5 + 0.25
    m1, s1 = np.mean(a.numpy(), axis=0), np.cov(a.numpy(), rowvar=False)
    m2, s2 = np.mean(b.numpy(), axis=0), np.cov(b.numpy(), rowvar=False)
    value = float(fid_score.calculate_frechet_distance(m1, s1, m2, s2))
    out["fd"] = {"x1": a, "x2": b, "value": value}
    print(f"calculate_frechet_distance {value:.12f}")

    real = os.path.join(torch.hub.get_dir(), "checkpoints", WEIGHT_FILE)
    if os.path.exists(real):
        rsd = torch.load(real, map_location="cpu")
        rnet = build_reference(inception, rsd)
        u8 = fo.image_bytes((256, 256), 31)[None]
        with torch.no_grad():
            ref = rnet(u8.permute(0, 3, 1, 2).contiguous().float().div(255))[0].flatten(1)
            ora = fo.forward({k: v.float() for k, v in rsd.items()}, fo.preprocess(u8))
        print(f"real weights ({len(rsd)} tensors): max|ref| {float(ref.abs().max()):.3f}, "
              f"oracle max|diff| {float((ora - ref).abs().max()):.2e}")
    else:
        print(f"{WEIGHT_FILE} is not in the torch hub cache: the oracle is checked on seeded weights only")
    torch.save(out, OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1e6:.2f} MB); worst oracle rel diff {worst:.2e}")


if __name__ == "__main__":
    main()
