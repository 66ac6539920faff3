"""CPU checks of the video-clip input side: the host twin of omt_resample_clips (layout.resize_clip with its fp32 axis
tables and single-rounding fma) equals the Latte loaders' torch pipeline bit for bit, live and through the golden fixture;
the geometry follows torch's shape rule and center_crop's rounding and errors; the flip draws consume Python's random as
RandomHorizontalFlipVideo does.  Floats are compared as int32 bit patterns."""
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from omnitokenizer_b200 import layout as L
from omnitokenizer_b200.consumers import LATTE_NORM
from oracle import make_golden_clips as G
from tests.util import load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PRESETS = {"ucf": L.ucf_clip_resize, "sky": L.sky_clip_resize, "taichi": lambda s: L.taichi_clip_resize()}
# (H, W) sources: UCF-101, portrait, 1080p, upscales from 1 x 1, odd sizes, short sides at the output size, and sizes
# whose scaled or cropped offsets are halves
SWEEP = [(240, 320), (320, 240), (1080, 1920), (1, 1), (2, 3), (37, 1000), (250, 333), (333, 250), (256, 455), (256, 341),
         (100, 130), (33, 33), (256, 256)]


def _bits(t):
    return t.contiguous().view(torch.int32)


def live_pipeline(clip, resize, flip, channels_last=True, norm=LATTE_NORM):
    """The loader's Compose restated with the same torch ops (video_transforms.py + torchvision Normalize) on a
    read_video-style (F, 3, H, W) view; channels_last=False makes the view contiguous first."""
    x = clip.permute(0, 3, 1, 2)
    if not channels_last:
        x = x.contiguous()
    x = x.float() / 255.0
    if flip:
        x = x.flip(-1)
    s = resize.size
    if resize.mode == "scale_crop":
        x = Fn.interpolate(x, scale_factor=s / min(x.shape[-2:]), mode="bilinear", align_corners=False)
        h, w = x.shape[-2:]
        if h < s or w < s:
            raise ValueError("height and width must be no smaller than crop_size")
        i, j = int(round((h - s) / 2.0)), int(round((w - s) / 2.0))
        x = x[..., i:i + s, j:j + s]
    elif resize.mode == "crop_resize":
        h, w = x.shape[-2:]
        if h < w:
            j = int(round((w - h) / 2.0))
            x = x[..., :, j:j + h]
        else:
            i = int(round((h - w) / 2.0))
            x = x[..., i:i + w, :]
        x = Fn.interpolate(x, size=(s, s), mode="bilinear", align_corners=False)
    mean = torch.as_tensor(norm.mean, dtype=torch.float32).view(-1, 1, 1)
    std = torch.as_tensor(norm.std, dtype=torch.float32).view(-1, 1, 1)
    return x.sub_(mean).div_(std)


def sweep_mismatches():
    """{case: mismatching outputs} of the host twin against live torch over the sweep, both thread modes, both input
    layouts, flip on and off, at output sizes on both sides of torch's 128-pixel kernel switch."""
    g = torch.Generator().manual_seed(1)
    threads = torch.get_num_threads()
    out = {}
    try:
        for H, W in SWEEP:
            clip = torch.randint(0, 256, (2, H, W, 3), generator=g, dtype=torch.uint8)
            for mode, s in (("scale_crop", 256), ("scale_crop", 40), ("crop_resize", 64), ("crop_resize", 200)):
                for in_workers in (True, False):
                    torch.set_num_threads(1 if in_workers else max(threads, 2))
                    rz = L.ClipResize(mode, s, True, in_workers)
                    for flip in (False, True):
                        try:
                            want = [live_pipeline(clip, rz, flip, cl) for cl in (True, False)]
                        except ValueError:
                            continue
                        got = _bits(L.resize_clip(clip, rz, flip, LATTE_NORM))
                        for cl, w in zip((True, False), want):
                            out[f"{H}x{W} {mode} {s} workers={in_workers} flip={flip} cl={cl}"] = int((got != _bits(w)).sum())
    finally:
        torch.set_num_threads(threads)
    return out


@pytest.mark.parametrize("capability", ["avx2", "avx512"])
def test_host_twin_equals_torch_under_each_dispatch(capability):
    """Each leg runs in a subprocess with ATEN_CPU_CAPABILITY set, where the host CPU supports it."""
    code = ("import json, torch; from tests import test_clip_ingest_cpu as t; "
            "print(json.dumps([torch.backends.cpu.get_cpu_capability(), t.sweep_mismatches()]))")
    env = dict(os.environ, ATEN_CPU_CAPABILITY=capability, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    got_cap, mism = json.loads(r.stdout.strip().splitlines()[-1])
    if got_cap.lower() != capability:
        pytest.skip(f"the host CPU does not run torch's {capability} kernels (got {got_cap})")
    assert len(mism) > 100
    assert not any(mism.values()), {k: v for k, v in mism.items() if v}


def test_host_twin_equals_torch_in_process():
    cap = torch.backends.cpu.get_cpu_capability()
    mism = sweep_mismatches()
    if cap == "DEFAULT":
        # without FMA, torch rounds every product and sum on its own: the documented difference, not an exact match
        assert sum(mism.values()) > 0
    else:
        assert not any(mism.values()), {k: v for k, v in mism.items() if v}


def test_default_capability_differs_as_documented():
    """Under ATEN_CPU_CAPABILITY=default torch takes scalar code without FMA; the twin follows the x86-64 FMA kernels."""
    code = ("import json, torch; from tests import test_clip_ingest_cpu as t; "
            "print(json.dumps([torch.backends.cpu.get_cpu_capability(), t.sweep_mismatches()]))")
    env = dict(os.environ, ATEN_CPU_CAPABILITY="default", PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    got_cap, mism = json.loads(r.stdout.strip().splitlines()[-1])
    assert got_cap == "DEFAULT"
    assert sum(mism.values()) > 0


def test_fma32_rounds_once():
    from fractions import Fraction
    g = np.random.default_rng(0)
    a, b, c = (g.random(20000).astype(np.float32) for _ in range(3))
    c[::2] *= np.float32(2.0 ** -30)            # addends far below the product: the fp64 sum is inexact
    got = L.fma32(a, b, c)
    for i in range(0, 20000, 37):
        assert got[i] == _round_f32(Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i])))
    # 4097 * 4097 = 2^24 + 2^13 + 1 lies exactly between two fp32 values, and +-2^-30 vanishes in the fp64 sum: only
    # the single rounding sends it up for a positive addend
    x = np.float32(4097)
    assert L.fma32(x, x, np.float32(2.0 ** -30)) == np.float32(16785410)
    assert L.fma32(x, x, np.float32(-2.0 ** -30)) == np.float32(16785408)
    assert L.fma32(x, x, np.float32(0)) == np.float32(16785408)


def _round_f32(v):
    """A Fraction rounded to the nearest fp32, ties to even."""
    from fractions import Fraction
    x = np.float32(float(v))
    cands = [np.nextafter(x, np.float32(-np.inf)), x, np.nextafter(x, np.float32(np.inf))]
    return min(cands, key=lambda c: (abs(Fraction(float(c)) - v), int(np.array(c).view(np.int32)) & 1))


def test_output_sizes_follow_torch():
    for H in range(1, 400, 7):
        for W in (1, 3, 240, 320, 341, 1000):
            for s in (32, 256):
                want = Fn.interpolate(torch.zeros(1, 1, H, W), scale_factor=s / min(H, W), mode="bilinear",
                                      align_corners=False).shape[-2:]
                assert L.scaled_size(H, W, s) == tuple(want)


def test_crop_offsets_round_half_to_even():
    g = L.clip_geometry(256, 341, L.ucf_clip_resize(256))
    assert (g.rh, g.rw, g.cy, g.cx) == (256, 341, 0, 42)            # 42.5 -> 42
    g = L.clip_geometry(256, 455, L.ucf_clip_resize(256))
    assert (g.rh, g.rw, g.cy, g.cx) == (256, 455, 0, 100)           # 99.5 -> 100
    g = L.clip_geometry(240, 321, L.sky_clip_resize(32))
    assert (g.y0, g.x0, g.wh, g.ww) == (0, 40, 240, 240)            # 40.5 -> 40
    g = L.clip_geometry(323, 240, L.sky_clip_resize(32))
    assert (g.y0, g.x0, g.wh, g.ww) == (42, 0, 240, 240)            # 41.5 -> 42
    g = L.clip_geometry(240, 320, L.ucf_clip_resize(256))
    assert (g.rh, g.rw, g.cy, g.cx) == (256, 341, 0, 42) and g.scale_h == g.scale_w == float(np.float32(240 / 256))


def test_raising_short_sides_match_torch():
    """UCFCenterCropVideo raises for the short sides whose scaled size floors to s - 1; the set matches torch's."""
    s = 256
    want = {n for n in range(1, 1001) if Fn.interpolate(torch.zeros(1, 1, n, n + 7, device="meta"), scale_factor=s / n,
                                                          mode="bilinear", align_corners=False).shape[-2] < s}
    got = set()
    for n in range(1, 1001):
        try:
            L.clip_geometry(n, n + 7, L.ucf_clip_resize(s))
        except ValueError as e:
            assert "no smaller than crop_size" in str(e)
            got.add(n)
    assert got == want and 49 in got and 239 in got and 240 not in got


def test_clip_params_draw_like_the_flip_transform():
    rz = L.ucf_clip_resize(32)
    random.seed(5)
    torch.manual_seed(0)
    t0 = torch.get_rng_state()
    want = [random.random() < 0.5 for _ in range(9)]
    st = random.getstate()
    random.seed(5)
    assert L.clip_params(9, rz) == want and random.getstate() == st
    assert torch.equal(torch.get_rng_state(), t0)
    random.seed(5)
    st = random.getstate()
    assert L.clip_params(4, L.sky_clip_resize(32)) == [False] * 4 and random.getstate() == st
    with pytest.raises(ValueError, match="not a draw"):
        L.check_clip_params([True], 1, L.sky_clip_resize(32))
    with pytest.raises(ValueError, match="2 clip parameters for 1"):
        L.check_clip_params([False, False], 1, rz)


def test_spec_checks():
    with pytest.raises(ValueError, match="mode"):
        L.check_clip_resize(L.ClipResize("zoom", 32))
    with pytest.raises(ValueError, match="size"):
        L.check_clip_resize(L.ClipResize("none", 32))
    with pytest.raises(TypeError):
        L.check_clip_resize(L.U8Resize((32, 32)))
    with pytest.raises(ValueError, match="largest byte"):
        L.clip_norm_table(L.U8Norm("v", (0.5,) * 3, (1.0,) * 3, max_test=True))
    t = L.clip_norm_table(LATTE_NORM)
    assert t.shape == (262,) and torch.equal(t[:256], torch.arange(256, dtype=torch.uint8).float() / 255.0)


@pytest.mark.parametrize("name", list(PRESETS))
def test_host_twin_equals_golden(name):
    fx = load_golden("clip_resize")
    srcs = G.sources(fx["taichi_sizes"] if name == "taichi" else fx["sizes"], fx["source_seed"], fx["frames"])
    assert [int(c.long().sum()) for c in srcs] == fx["source_sum"][name]
    rz = PRESETS[name](fx["s"])
    random.seed(fx["seed"])
    flips = L.clip_params(len(srcs), rz)
    assert flips == fx[name]["flips"] and random.getstate() == fx[name]["random_after"]
    for c, f, want in zip(srcs, flips, fx[name]["out"]):
        assert torch.equal(_bits(L.resize_clip(c, rz, f, LATTE_NORM)), _bits(want)), (name, tuple(c.shape))
    assert fx["num_threads"] == 1 and isinstance(fx["cpu_capability"], str)


def test_golden_fixture_reproduced():
    from oracle import ref_loader
    if not ref_loader.available():
        pytest.skip("the reference tree is not present")
    pytest.importorskip("torchvision")
    want = load_golden("clip_resize")
    got = G.build(want["s"], want["seed"])
    for k in ("sizes", "taichi_sizes", "source_sum", "frames", "num_threads", "cpu_capability"):
        assert got[k] == want[k], k
    for name in PRESETS:
        assert got[name]["flips"] == want[name]["flips"] and got[name]["random_after"] == want[name]["random_after"]
        for a, b in zip(got[name]["out"], want[name]["out"]):
            assert torch.equal(_bits(a), _bits(b))


def test_consumer_transforms_on_the_host_for_other_models():
    """A model without encode_clips_u8 gets latte_encode_latents of the host pipeline's fp32 clips."""
    from omnitokenizer_b200 import consumers as C

    class Fake:
        def __init__(self):
            self.seen = []

        def encode(self, x, is_image, include_embeddings=False):
            self.seen.append((x.clone(), is_image))
            return torch.ones(x.shape[0], 4, 1 + (x.shape[2] - 1) // 4, 2, 2)

    g = torch.Generator().manual_seed(9)
    clips = [torch.randint(0, 256, (5, h, w, 3), generator=g, dtype=torch.uint8) for h, w in ((24, 40), (40, 33), (32, 32))]
    rz = L.ucf_clip_resize(32)
    fake = Fake()
    random.seed(2)
    z = C.latte_encode_latents_clips_u8(fake, clips, rz)
    random.seed(2)
    flips = L.clip_params(3, rz)
    want = torch.stack([L.resize_clip(c, rz, f, LATTE_NORM) for c, f in zip(clips, flips)]).permute(0, 2, 1, 3, 4)
    x, is_image = fake.seen[0]
    assert torch.equal(_bits(x), _bits(want)) and not is_image
    assert torch.equal(z, torch.full((3, 2, 4, 2, 2), C.LATENT_SCALE))
