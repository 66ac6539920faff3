"""Generate tests/golden/fvd_suite.pt from the UNMODIFIED reference video-metric suite
(evaluation/common_metrics_on_video_quality: calculate_fvd.py, fvd/styleganv/fvd.py with its i3d_torchscript.pt,
fvd/videogpt/fvd.py with its pytorch_i3d.py), loaded by file path and run on the CPU.

- preprocess: SHA-256 of each method's get_fvd_feats input (styleganv preprocess_single per clip, videogpt
  preprocess) for seeded fp32 clips of several sizes, grey included;
- seeded: the torchscript with seeded weights (i3d_oracle.make_state_dict + calibrate_bn, under its key names) and
  its features of three clips; the oracle's forward is checked against it;
- shipped: the torchscript's own weights on two clips (features only; the weights are not stored);
- fvd: calculate_fvd's dicts of both methods on 8 + 8 clips of 12 frames at 64 x 64 (bytes / 255), each network
  replaced by its seeded weights (videogpt: tests/golden/fvd_i3d.pt's).  videogpt's features are widened to float64
  before its frechet_distance, as this project's calculate_fvd does, so the distance is not fp32 noise.

    python -m oracle.make_golden_fvd_suite
"""
import hashlib
import importlib.util
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import fvd_suite_oracle as so  # noqa: E402
from oracle import i3d_oracle as io  # noqa: E402
from oracle.ref_loader import REF_ROOT  # noqa: E402
from omnitokenizer_b200 import quality  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "fvd_suite.pt")
SUITE = os.path.join(REF_ROOT, "evaluation", "common_metrics_on_video_quality")
TORCHSCRIPT = os.path.join(SUITE, "fvd", "styleganv", "i3d_torchscript.pt")
# (name, (B, T, C, H, W), seed): fp32 clips of torch.rand, off the byte grid
PRE_CASES = [("64", (2, 10, 3, 64, 64), 1), ("128", (1, 10, 3, 128, 128), 2), ("256", (1, 10, 3, 256, 256), 3),
             ("240x320", (1, 10, 3, 240, 320), 4), ("320x240", (1, 10, 3, 320, 240), 5),
             ("97x131", (1, 11, 3, 97, 131), 6), ("grey_80x96", (1, 10, 1, 80, 96), 7)]
FEAT_CASES = [("64", (1, 10, 3, 64, 64), 21), ("97x131", (1, 11, 3, 97, 131), 22), ("grey_80x96", (1, 10, 1, 80, 96), 23)]
SHIPPED_CASE = ("shipped_2x10x64", (2, 10, 3, 64, 64), 31)
SGV_SEED = 9
FVD_SET = (8, 12, 64, 64)        # clips per side, frames, H, W
FVD_SEED = 41


def clips(shape, seed):
    return torch.rand(shape, generator=torch.Generator().manual_seed(seed))


def fvd_sets():
    """gt and gen uint8 (B, T, H, W, 3): gen is a shifted, dimmed copy of gt (close, not equal)."""
    B, T, H, W = FVD_SET
    gt = torch.randint(0, 256, (B, T, H, W, 3), generator=torch.Generator().manual_seed(FVD_SEED), dtype=torch.uint8)
    gen = gt.clone()
    gen[..., 1:, :] = gen[..., :-1, :]
    return gt, (gen.int() * 7 // 8 + 16).to(torch.uint8)


def u8_to_f32(u8):
    return u8.float().permute(0, 1, 4, 2, 3).contiguous() / 255.


def sha(t: torch.Tensor) -> str:
    return hashlib.sha256(t.contiguous().numpy().tobytes()).hexdigest()


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def load_reference():
    """The suite's calculate_fvd and both fvd modules under their package names (the package __init__, which imports
    the lpips package, is not run)."""
    for pkg, path in (("common_metrics_on_video_quality", SUITE), ("common_metrics_on_video_quality.fvd",
                                                                  os.path.join(SUITE, "fvd"))):
        m = types.ModuleType(pkg)
        m.__path__ = [path]
        sys.modules[pkg] = m
    for sub in ("styleganv", "videogpt"):
        m = types.ModuleType(f"common_metrics_on_video_quality.fvd.{sub}")
        m.__path__ = [os.path.join(SUITE, "fvd", sub)]
        sys.modules[m.__name__] = m
    sg = _load("common_metrics_on_video_quality.fvd.styleganv.fvd", os.path.join(SUITE, "fvd", "styleganv", "fvd.py"))
    vg = _load("common_metrics_on_video_quality.fvd.videogpt.fvd", os.path.join(SUITE, "fvd", "videogpt", "fvd.py"))
    pi3d = _load("common_metrics_on_video_quality.fvd.videogpt.pytorch_i3d",
                 os.path.join(SUITE, "fvd", "videogpt", "pytorch_i3d.py"))
    cf = _load("common_metrics_on_video_quality.calculate_fvd", os.path.join(SUITE, "calculate_fvd.py"))
    return cf, sg, vg, pi3d


def seeded_styleganv(first_clip):
    """i3d_oracle.make_state_dict(SGV_SEED) with BatchNorm calibrated on first_clip's network input, under the
    torchscript's keys, and the torchscript holding it."""
    sd = io.make_state_dict(SGV_SEED)
    io.calibrate_bn(sd, first_clip)
    net = torch.jit.load(TORCHSCRIPT).eval()
    missing, unexpected = net.load_state_dict(so.styleganv_keys(sd), strict=False)
    assert not unexpected and all(k.endswith("num_batches_tracked") for k in missing), (missing, unexpected)
    return sd, net


def main():
    cf, sg, vg, pi3d = load_reference()
    out = {"preprocess": {}, "feats": {}}
    # 1. preprocess hashes: the exact tensors each get_fvd_feats hands its network
    for name, shape, seed in PRE_CASES:
        v = clips(shape, seed)
        T = shape[1]
        x_sg = torch.stack([sg.preprocess_single(c) for c in cf.trans(v)])
        with so.threads_at_least(2):
            x_vg = vg.preprocess(cf.trans(v))
        assert torch.equal(x_sg, so.preprocess_styleganv(v, T)), name
        assert torch.equal(x_vg, so.preprocess_videogpt(v, T)), name
        out["preprocess"][name] = {"shape": shape, "seed": seed, "styleganv": sha(x_sg), "videogpt": sha(x_vg)}
    # 2. seeded weights in the live torchscript
    name0, shape0, seed0 = FEAT_CASES[0]
    sd, net = seeded_styleganv(so.preprocess_styleganv(clips(shape0, seed0), shape0[1]))
    out["sgv_seed"], out["sgv_bn"] = SGV_SEED, io.bn_stats(sd)
    worst = 0.0
    with torch.no_grad():
        for name, shape, seed in FEAT_CASES:
            v = clips(shape, seed)
            f = torch.from_numpy(sg.get_fvd_feats(cf.trans(v), net, "cpu")).float()
            o = so.forward_styleganv(net.state_dict(), so.preprocess_styleganv(v, shape[1]))
            worst = max(worst, float((f - o).abs().max() / f.abs().max()))
            out["feats"][name] = {"shape": shape, "seed": seed, "feats": f}
        # 3. the shipped weights
        shipped = torch.jit.load(TORCHSCRIPT).eval()
        name, shape, seed = SHIPPED_CASE
        v = clips(shape, seed)
        out["shipped"] = {"shape": shape, "seed": seed,
                          "feats": torch.from_numpy(sg.get_fvd_feats(cf.trans(v), shipped, "cpu")).float()}
    print(f"oracle vs torchscript (seeded): {worst:.2e} of max|feature|")
    # 4. calculate_fvd of both methods
    gt, gen = fvd_sets()
    vsd = io.make_state_dict(torch.load(os.path.join(ROOT, "tests", "golden", "fvd_i3d.pt"))["w_seed"])
    vsd.update(torch.load(os.path.join(ROOT, "tests", "golden", "fvd_i3d.pt"))["bn"])
    vnet = pi3d.InceptionI3d(400, in_channels=3).eval()
    vnet.load_state_dict(vsd)
    sg.load_i3d_pretrained = lambda device=None: net
    sg.sqrtm = quality.sqrtm_disp                # scipy >= 1.16 dropped sqrtm's disp argument the module passes
    vg.load_i3d_pretrained = lambda device=None: vnet
    logits = vg.get_fvd_logits
    vg.get_fvd_logits = lambda videos, i3d, device, bs=10: logits(videos, i3d, device, bs).double()
    out["fvd"] = {"set": FVD_SET, "seed": FVD_SEED}
    with torch.no_grad(), so.threads_at_least(2):
        for method in ("styleganv", "videogpt"):
            r = cf.calculate_fvd(u8_to_f32(gt), u8_to_f32(gen), "cpu", method=method)
            out["fvd"][method] = {"value": {int(k): float(v) for k, v in r["value"].items()},
                                  "video_setting": tuple(r["video_setting"]),
                                  "video_setting_name": r["video_setting_name"]}
            print(method, out["fvd"][method]["value"])
    torch.save(out, OUT)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
