"""The suite's AlexNet LPIPS without a GPU: the oracle through the suite's loop against the fixture, the wiring breaks
the fixture detects, the tap sizes against torchvision, both weight layouts and conv1's packing, the named key errors
and every refusal of quality.AlexLPIPS / calculate_lpips before a launch."""
import os

import numpy as np
import pytest
import torch

from omnitokenizer_b200 import quality
from oracle import lpips_alex_oracle as ao

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "lpips_alex.pt")
LPIPS_REL = 1e-4                    # the GPU path's per-frame tolerance (tests/test_gpu_lpips_alex.py)


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN)


@pytest.fixture(scope="module")
def sd(golden):
    sd = ao.make_state_dict(golden["w_seed"])
    assert ao.fingerprint(sd) == golden["fingerprint"]
    return sd


def _per_frame(net, spec):
    v1, v2 = ao.videos(spec)
    with torch.no_grad():
        return ao.suite_loop(net, v1, v2, torch.device("cpu"))


def _rel(got, want):
    return float(((got - want).abs() / want.abs().clamp_min(1e-30)).max())


def test_oracle_reproduces_fixture(golden, sd):
    net = ao.AlexLPIPSOracle(sd).eval()
    for name, e in golden["cases"].items():
        net.maps = [] if name == golden["maps_case"] else None
        per = _per_frame(net, e["spec"])
        B, T, C, H, W = e["spec"][:5]
        if name.startswith("same"):
            assert bool((per == 0).all()) and bool((e["per_frame"] == 0).all()), name
        else:
            assert _rel(per, e["per_frame"]) <= 1e-6, name
        r = quality.result_dict(e["per_frame"].numpy(), torch.Size([T, 3, H, W]))
        assert r["video_setting"] == torch.Size(e["video_setting"]) and r["video_setting_name"] == e["video_setting_name"]
        for t in range(T):
            assert r["value"][t] == e["value"][t] and r["value_std"][t] == e["value_std"][t], name
        if net.maps is not None:
            taps, val = net.maps[0]
            for got, want in zip(taps, e["tap_maps"]):
                assert torch.allclose(got[0, 0], want, rtol=1e-5, atol=1e-9)
            assert torch.allclose(val[0, 0], e["map"], rtol=1e-5, atol=1e-9)


BREAKS = [dict(align_corners=True), dict(spatial_average=True), dict(scaling=False), dict(pre_relu=True),
          dict(drop_tap=4), dict(eps=0.1)]


@pytest.mark.parametrize("kw", BREAKS, ids=[next(iter(k)) for k in BREAKS])
def test_wiring_breaks_are_detected(golden, sd, kw):
    """Each broken wiring moves some case's frame value, or the stored spatial map, by more than 100 times the GPU
    tolerance.  (The bilinear upsample with half-pixel centres nearly keeps a map's mean, so the spatial average moves
    the frame values by about 3e-4 only; it changes the map itself.)"""
    net = ao.AlexLPIPSOracle(sd, **kw).eval()
    worst = 0.0
    for name in ("min_31x45", "bytes_67x93", "border_64", "demo_zeros_ones_64"):
        e = golden["cases"][name]
        net.maps = [] if name == golden["maps_case"] else None
        worst = max(worst, _rel(_per_frame(net, e["spec"]), e["per_frame"]))
        if net.maps is not None:
            val = net.maps[0][1][0, 0].expand_as(e["map"])
            worst = max(worst, float((val - e["map"]).abs().max() / e["map"].abs().max()))
    print(f"{kw}: worst rel {worst:.1e}")
    assert worst > 100 * LPIPS_REL


def test_tap_sizes_against_torchvision():
    import torchvision
    feats = torchvision.models.alexnet(weights=None).features.to("meta")
    for H in range(31, 301):
        W = 331 - H
        x = torch.empty(1, 3, H, W, device="meta")
        got = []
        for a, b in ao.SLICE_BOUNDS:
            for i in range(a, b):
                x = feats[i](x)
            got.append(tuple(x.shape[2:]))
        assert quality.alex_tap_sizes(H, W) == got, (H, W)
    assert quality.alex_tap_sizes(64, 64)[0] == (15, 15) and quality.alex_tap_sizes(256, 256)[2] == (15, 15)
    for H, W in ((30, 64), (64, 30), (30, 30)):
        with pytest.raises(ValueError, match="31"):
            quality.alex_tap_sizes(H, W)
        with pytest.raises(RuntimeError):
            feats(torch.empty(1, 3, H, W, device="meta"))


def _planes(m):
    return [u.w_hi + u.w_lo for u in m.convs]


def test_layouts_load_the_same_planes(sd, tmp_path):
    bare = quality.AlexLPIPS(sd, device="cpu")
    tv = ao.torchvision_state_dict(sd)
    tv["classifier.1.weight"] = torch.zeros(4096, 9216)
    lin = {k: v for k, v in sd.items() if k.startswith("lin")}
    from_tv = quality.AlexLPIPS({**tv, **lin}, device="cpu")
    torch.save(tv, tmp_path / "alexnet.pth")
    torch.save(lin, tmp_path / "alex.pth")
    from_files = quality.load_lpips_alex("cpu", str(tmp_path / "alexnet.pth"), str(tmp_path / "alex.pth"))
    no_scaling = quality.AlexLPIPS({k: v for k, v in sd.items() if not k.startswith("scaling_layer")}, device="cpu")
    for m in (from_tv, from_files, no_scaling):
        assert all(torch.equal(x, y) for x, y in zip(_planes(m), _planes(bare)))
        assert all(torch.equal(x, y) for x, y in zip(m.lin, bare.lin))
        assert torch.equal(m.shift_scale, bare.shift_scale)
    sd2 = dict(sd)
    sd2["scaling_layer.scale"] = sd["scaling_layer.scale"] * 2
    assert not torch.equal(quality.AlexLPIPS(sd2, device="cpu").shift_scale, bare.shift_scale)
    # conv1: K = (dh, dw, c) over 11 x 11 taps of the 4-channel input, 484 rounded up to 512, cout padded to 128
    u = bare.convs[0]
    assert u.K == 512 and u.w_hi.shape == (128, 512) and u.k == (1, 11, 11) and u.stride == (1, 4, 4)
    packed = u.w_hi + u.w_lo
    w = sd["net.slice1.0.weight"]
    assert torch.equal(packed[:64, :484].view(64, 11, 11, 4)[..., :3], w.permute(0, 2, 3, 1))
    assert not bool(packed[:64, :484].view(64, 11, 11, 4)[..., 3].any()) and not bool(packed[:, 484:].any())
    assert not bool(packed[64:].any())
    for m, c in zip(bare.convs, quality.ALEX):
        assert m.K == c.k * c.k * c.cin if c.cin > 3 else True
        assert m.k == (1, c.k, c.k) and m.stride == (1, c.stride, c.stride) and m.cout == c.cout


def test_named_key_errors(sd):
    bad = dict(sd)
    del bad["lin2.model.1.weight"]
    with pytest.raises(KeyError, match="lin2.model.1.weight"):
        quality.AlexLPIPS(bad, device="cpu")
    bad = dict(sd)
    bad["net.slice2.3.weight"] = torch.zeros(192, 64, 3, 3)
    with pytest.raises(ValueError, match=r"net\.slice2\.3\.weight"):
        quality.AlexLPIPS(bad, device="cpu")
    tv = {**ao.torchvision_state_dict(sd), "features.12.weight": torch.zeros(1)}
    with pytest.raises(KeyError, match="features.12"):
        quality.AlexLPIPS(tv, device="cpu")
    bad = dict(sd)
    bad["net.slice6.12.weight"] = torch.zeros(1)
    with pytest.raises(KeyError, match="slice6"):
        quality.AlexLPIPS(bad, device="cpu")


def test_other_options_refused(sd):
    with pytest.raises(NotImplementedError, match="squeeze"):
        quality.AlexLPIPS(sd, device="cpu", net="squeeze")
    with pytest.raises(NotImplementedError, match="spatial"):
        quality.AlexLPIPS(sd, device="cpu", spatial=False)
    with pytest.raises(NotImplementedError, match="AlexLPIPS"):
        quality.LPIPS(quality.lpips_state_dict({}), device="cpu", net="alex")


def _f(*shape, dtype=torch.float32):
    return torch.zeros(*shape, dtype=dtype)


@pytest.mark.parametrize("case,exc,match", [
    ((_f(1, 2, 3, 64, 64), _f(1, 2, 3, 64, 65)), ValueError, "differ in shape"),
    ((_f(1, 2, 3, 30, 64), _f(1, 2, 3, 30, 64)), ValueError, "31"),
    ((_f(1, 2, 3, 64, 30), _f(1, 2, 3, 64, 30)), ValueError, "31"),
    ((_f(1, 2, 64, 64, 3, dtype=torch.uint8), _f(1, 2, 64, 64, 3, dtype=torch.uint8)[..., :30, :]), ValueError,
     "differ in shape"),
    ((_f(1, 2, 3, 64, 64, dtype=torch.float64), _f(1, 2, 3, 64, 64, dtype=torch.float64)), TypeError, "float64"),
    ((_f(1, 2, 3, 64, 64), _f(1, 2, 64, 64, 3, dtype=torch.uint8)), TypeError, "uint8"),
    ((_f(2, 3, 64, 64), _f(2, 3, 64, 64)), ValueError, r"\(B, T, C, H, W\)"),
    ((_f(1, 2, 2, 64, 64), _f(1, 2, 2, 64, 64)), ValueError, "C 1 or 3"),
    ((_f(1, 2, 64, 64, 1, dtype=torch.uint8), _f(1, 2, 64, 64, 1, dtype=torch.uint8)), ValueError, r"H, W, 3"),
    ((_f(0, 2, 3, 64, 64), _f(0, 2, 3, 64, 64)), ValueError, "empty"),
    ((np.zeros((1, 2, 3, 64, 64), np.float32), _f(1, 2, 3, 64, 64)), TypeError, "torch tensor"),
], ids=["shape", "small_h", "small_w", "u8_shape", "float64", "mixed", "rank", "channels", "u8_channels", "empty",
        "numpy"])
def test_calculate_lpips_refusals(sd, case, exc, match):
    m = quality.AlexLPIPS(sd, device="cpu")
    with pytest.raises(exc, match=match):
        quality.calculate_lpips(*case, device="cpu", model=m)


def test_calculate_lpips_device_refusals(sd):
    m = quality.AlexLPIPS(sd, device="cpu")
    v = _f(1, 2, 3, 64, 64)
    with pytest.raises(ValueError, match="CUDA"):
        quality.calculate_lpips(v, v, "cpu", model=m)
    with pytest.raises(ValueError, match="is on cpu"):
        quality.calculate_lpips(v, v, "cuda:1", model=m)
    with pytest.raises(TypeError, match="load_lpips_alex"):
        quality.calculate_lpips(v, v, "cuda:0")
    with pytest.raises(TypeError, match="load_lpips_alex"):
        quality.calculate_lpips(v, v, "cuda:0", model=quality.LPIPS.__new__(quality.LPIPS))
