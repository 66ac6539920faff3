"""The suite's AlexNet LPIPS on the GPU: omt_lpips_map against fp64 and against omt_lpips_head, omt_lpips_upsample_mean
bit for bit against torch's CUDA bilinear upsample, calculate_lpips end to end against the fixture, the uint8 / grey /
chunked / graphed forms bit for bit, and omt_conv3d's error at AlexNet's conv geometries.  Measured worst cases are
printed."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from omnitokenizer_b200 import _cabi, quality
from oracle import lpips_alex_oracle as ao
from tests import conv_cases as cc

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "lpips_alex.pt")
LPIPS_REL = 1e-4                    # per frame, relative: the VGG LPIPS bound (test_gpu_quality.py)


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN)


@pytest.fixture(scope="module")
def model(golden):
    sd = ao.make_state_dict(golden["w_seed"])
    assert ao.fingerprint(sd) == golden["fingerprint"]
    return quality.AlexLPIPS(sd, DEV)


def _features(C, Cs, h, w, P, seed):
    """Post-ReLU features [2P][h][w][Cs]; the Cs - C padding channels hold large values the kernels must not read."""
    g = torch.Generator().manual_seed(seed)
    x = torch.full((2 * P, h, w, Cs), 1e6)
    x[..., :C] = torch.relu(torch.randn(2 * P, h, w, C, generator=g))
    x[0, 0, 0, :C] = 0                               # an all-zero feature vector: normalises to zero via the 1e-10
    return x, torch.rand(C, generator=g)


@pytest.mark.parametrize("C,Cs,h,w,P", [(64, 64, 15, 15, 3), (192, 192, 7, 10, 2), (384, 384, 3, 4, 4),
                                        (256, 256, 1, 1, 5), (256, 256, 63, 63, 2), (64, 96, 15, 15, 3),
                                        (192, 224, 7, 10, 2), (40, 64, 5, 6, 2)])
def test_lpips_map_against_fp64_and_head(C, Cs, h, w, P):
    x, lin = _features(C, Cs, h, w, P, C + Cs + h)
    xd, lind = x.to(DEV), lin.to(DEV)
    m = torch.full((P, h, w), -1.0, device=DEV)
    _cabi.call("omt_lpips_map", xd, Cs, C, P, h, w, lind, m)
    taps = torch.zeros(5, P, device=DEV)
    _cabi.call("omt_lpips_head", xd, Cs, C, P, h, w, lind, 1, taps, None)
    torch.cuda.synchronize()
    xa, xb = x[:P, ..., :C].double(), x[P:, ..., :C].double()
    na = xa / (xa.pow(2).sum(-1, keepdim=True).sqrt() + 1e-10)
    nb = xb / (xb.pow(2).sum(-1, keepdim=True).sqrt() + 1e-10)
    ref = ((na - nb) ** 2 * lin.double()).sum(-1)
    got = m.cpu().double()
    rel = float(((got - ref).abs() / ref.abs().clamp_min(1e-30)).max())
    # the head sums exactly these pixels, but in another fp64 order: its value is within 1 ulp of the map's fp64 mean
    mean64 = got.flatten(1).sum(1) / (h * w)
    head = taps[1].cpu()
    exact = int((mean64.float() == head).sum())
    ulps = float(((mean64.float() - head).abs() / torch.from_numpy(np.spacing(head.numpy()))).max())
    print(f"map C={C} of {Cs} {h}x{w}: rel {rel:.1e}; head = fp64 mean of the map in {exact}/{P} pairs, "
          f"worst {ulps:.0f} ulp")
    assert rel <= 2e-6
    assert ulps <= 1


def _torch_spatial(maps, H, W):
    """lpips.py's spatial tail on torch's CUDA kernel: val = 0; val += upsample(res[k]) in order."""
    val = 0
    for m in maps:
        val += F.interpolate(m[:, None], size=(H, W), mode="bilinear", align_corners=False)
    return val[:, 0]


def _upsample_mean(maps, H, W, with_map=True):
    P = maps[0].shape[0]
    out = torch.full((P, H, W), -1.0, device=DEV) if with_map else None
    mean = torch.full((P,), -1.0, device=DEV)
    taps = _cabi.lpips_taps([(m, m.shape[1], m.shape[2]) for m in maps])
    _cabi.call("omt_lpips_upsample_mean", taps, len(maps), P, H, W, out, mean)
    torch.cuda.synchronize()
    return out, mean


def _ulps(a, b):
    ia, ib = a.view(torch.int32).long(), b.view(torch.int32).long()
    ia = torch.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = torch.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return int((ia - ib).abs().max())


UP_CASES = [((31, 31), None), ((64, 64), None), ((67, 93), None), ((256, 256), None), ((512, 512), None),
            ((40, 52), [(1, 1), (40, 52), (7, 9), (40, 1), (2, 52)])]


@pytest.mark.parametrize("HW,sizes", UP_CASES, ids=["31", "64", "67x93", "256", "512", "1x1_and_full"])
def test_upsample_bit_equal_to_torch(HW, sizes):
    H, W = HW
    sizes = sizes or quality.alex_tap_sizes(H, W)
    g = torch.Generator().manual_seed(H * 1000 + W)
    P = 3
    maps = [(torch.rand(P, h, w, generator=g) * 10 ** float(k - 2)).to(DEV) for k, (h, w) in enumerate(sizes)]
    out, mean = _upsample_mean(maps, H, W)
    ref = _torch_spatial(maps, H, W)
    ulps = _ulps(out, ref)
    print(f"{H}x{W} taps {sizes}: {ulps} ulp from torch's CUDA upsample")
    assert ulps == 0, f"the map is {ulps} ulp from torch's upsample_bilinear2d"
    ref64 = ref.double().flatten(1).mean(1).cpu()
    half_ulp = torch.from_numpy(np.spacing(ref64.float().numpy())).double() / 2
    err = (mean.cpu().double() - ref64).abs()
    print(f"  mean: {float((err / half_ulp).max()):.2f} half-ulps from the fp64 mean")
    assert bool((err <= half_ulp * 1.0001).all())
    _, mean2 = _upsample_mean(maps, H, W, with_map=False)
    assert torch.equal(mean, mean2)


def test_upsample_refusals():
    m = torch.zeros(2, 3, 3, device=DEV)
    mean = torch.full((2,), -1.0, device=DEV)
    for taps, n, match in (([(m, 3, 3)] * 6, 6, "taps"), ([(None, 3, 3)], 1, "null map"), ([(m, 0, 3)], 1, "0x3"),
                           ([(m.data_ptr() + 2, 3, 3)], 1, "misaligned")):
        with pytest.raises(RuntimeError, match=match):
            _cabi.call("omt_lpips_upsample_mean", _cabi.lpips_taps(taps), n, 2, 8, 8, None, mean)
    with pytest.raises(RuntimeError, match="null pointer"):
        _cabi.call("omt_lpips_upsample_mean", _cabi.lpips_taps([(m, 3, 3)]), 1, 2, 8, 8, None, None)
    torch.cuda.synchronize()
    assert bool((mean == -1).all())


def test_fixture_end_to_end(golden, model):
    worst = 0.0
    for name, e in golden["cases"].items():
        v1, v2 = ao.videos(e["spec"])
        per = quality.lpips_alex_frames(v1, v2, DEV, model).cpu().double()
        want = e["per_frame"]
        if name.startswith("same"):
            assert bool((per == 0).all()), name
            continue
        rel = float(((per - want).abs() / want.abs()).max())
        worst = max(worst, rel)
        print(f"{name}: worst frame rel {rel:.1e}")
        assert rel <= LPIPS_REL, name
        r = quality.calculate_lpips(v1, v2, DEV, model)
        assert r["video_setting"] == torch.Size(e["video_setting"])
        for t, v in e["value"].items():
            assert abs(r["value"][t] - v) <= LPIPS_REL * abs(v), name
    print(f"fixture: worst frame rel {worst:.1e} (bound {LPIPS_REL:.0e})")


def test_u8_and_grey_forms_bit_equal(golden, model):
    e = golden["cases"]["bytes_67x93"]
    v1, v2 = ao.videos(e["spec"])
    f32 = quality.lpips_alex_frames(v1, v2, DEV, model)
    u8 = quality.lpips_alex_frames(ao.to_u8(v1).to(DEV), ao.to_u8(v2).to(DEV), DEV, model)
    assert torch.equal(f32, u8)
    g1, g2 = ao.videos(golden["cases"]["grey_64"]["spec"])
    grey = quality.lpips_alex_frames(g1.to(DEV), g2.to(DEV), DEV, model)
    rgb = quality.lpips_alex_frames(g1.repeat(1, 1, 3, 1, 1), g2.repeat(1, 1, 3, 1, 1), DEV, model)
    assert torch.equal(grey, rgb)


def test_chunked_equals_unchunked(model, monkeypatch):
    v1, v2 = ao.videos((3, 5, 3, 64, 48, "bytes", 21))
    whole = quality.lpips_alex_frames(v1, v2, DEV, model)
    monkeypatch.setattr(quality, "LPIPS_ROWS", 2 * 4 * 64 * 48)          # chunks of 4 pairs: 4, 4, 4, 3
    assert quality.chunk_pairs(15, 64, 48, True) == 4
    chunked = quality.lpips_alex_frames(v1, v2, DEV, model)
    assert torch.equal(whole, chunked)


def test_graph_replay_equals_eager(model):
    v1, v2 = ao.videos((2, 3, 3, 72, 56, "bytes", 22))
    outs = [quality.lpips_alex_frames(v1, v2, DEV, model).clone() for _ in range(3)]    # eager, capture, replay
    assert all(torch.equal(o, outs[0]) for o in outs[1:])
    ws = model._ws[(DEV, quality.FORM_F32, 6, 72, 56)]
    assert isinstance(ws.graphs.get("lpips_alex"), tuple)


ALEX_CASES = [cc._conv2d_case(f"alex{c.idx}", c.cin, c.cout, c.k, c.k, c.stride, c.pad, c.pad,
                              (67, 63) if c.idx == 0 else (13, 11), 0, c.cout, B=2) for c in quality.ALEX]


@pytest.mark.parametrize("c", ALEX_CASES, ids=[c.id for c in ALEX_CASES])
def test_alexnet_conv_geometry_against_fp64(c):
    x, w, b = cc.realistic_operands(c, 31)
    w_hi, w_lo = cc.pack(w, c)
    y = torch.full((c.M, c.ldy), float("nan"), device=DEV)
    _cabi.call("omt_conv3d", cc.to_cl(x, c.Cs).to(DEV), c.Cs, c.B, *c.dims, w_hi.to(DEV), w_lo.to(DEV), c.K, b.to(DEV),
               c.cout, *c.k, *c.s, *c.front, *c.out, y, c.ldy, 0)
    torch.cuda.synchronize()
    xd, wd, bd = x.to(DEV), w.to(DEV), b.to(DEV)
    err = cc.l2_error(y.view(c.B, *c.out, c.cout), cc.conv64(xd, wd, c, bd), cc.l2_scale(xd, wd, bd, c))
    print(f"{c.id}: {err:.2e} of the l2 norm")
    assert err <= cc.L2_BOUND, err


def test_oracle_on_gpu_matches_fixture(golden):
    """The restatement itself on the GPU in strict fp32 (no TF32): the suite's loop within the GPU tolerance."""
    sd = ao.make_state_dict(golden["w_seed"])
    net = ao.AlexLPIPSOracle(sd).eval().to(DEV)
    e = golden["cases"]["bytes_64"]
    v1, v2 = ao.videos(e["spec"])
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            per = ao.suite_loop(net, v1, v2, DEV)
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    assert float(((per - e["per_frame"]).abs() / e["per_frame"]).max()) <= LPIPS_REL
