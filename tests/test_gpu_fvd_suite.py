"""The video-metric suite's FVD on the GPU: omt_fvd_suite_preprocess against the oracle bit for bit, the StyleGAN-V
features against the live reference's (tests/golden/fvd_suite.pt), calculate_fvd against the reference's dicts, and
the prefix, chunk and graph invariances."""
import os

import pytest
import torch

from omnitokenizer_b200 import _cabi, consumers, fvd, quality
from omnitokenizer_b200.engine import CLIP_DESC_WORDS
from oracle import fvd_suite_oracle as so
from oracle import i3d_oracle as io

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
HERE = os.path.dirname(__file__)
GOLDEN = os.path.join(HERE, "golden", "fvd_suite.pt")
SHIPPED = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "i3d_styleganv.pt")


def rand(shape, seed):
    return torch.rand(shape, generator=torch.Generator().manual_seed(seed))


def u8(shape, seed):
    return torch.randint(0, 256, shape, generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)


def device_preprocess(src, form, t):
    """omt_fvd_suite_preprocess of the first t frames of every clip -> (B, 3, t, 224, 224) on the host."""
    c = fvd.SuiteClips(src.to(DEV).contiguous(), form)
    out = torch.full((c.B, t, 224, 224, 4), float("nan"), device=DEV)
    _cabi.call("omt_fvd_suite_preprocess", c.src, c.src.numel(), form, c.C, c.desc, c.desc_host, c.tab, c.tab_host,
               c.tab_host.numel(), c.B, t, 224, 224, out)
    torch.cuda.synchronize()
    assert bool((out[..., 3] == 0).all())
    return out[..., :3].permute(0, 4, 1, 2, 3).cpu()


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN)


@pytest.fixture(scope="module")
def sgv(golden):
    sd = io.make_state_dict(golden["sgv_seed"])
    sd.update(golden["sgv_bn"])
    return fvd.load_i3d_styleganv(DEV, so.styleganv_keys(sd))


@pytest.fixture(scope="module")
def vgpt():
    g = torch.load(os.path.join(HERE, "golden", "fvd_i3d.pt"))
    sd = io.make_state_dict(g["w_seed"])
    sd.update(g["bn"])
    return fvd.I3D(sd, DEV)


SHAPES = [(2, 10, 3, 64, 64), (1, 10, 3, 128, 128), (1, 10, 3, 256, 256), (1, 10, 3, 240, 320), (1, 10, 3, 320, 240),
          (1, 11, 3, 97, 131), (1, 10, 1, 80, 96)]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("method", ["styleganv", "videogpt"])
def test_preprocess_matches_oracle(shape, method):
    v = rand(shape, 100 + shape[-1])                      # off the byte grid: the videogpt truncation matters
    form = fvd.FORM_F32 if method == "styleganv" else fvd.FORM_F32_TRUNC
    fn = so.preprocess_styleganv if method == "styleganv" else so.preprocess_videogpt
    for t in (10, shape[1]):
        got, want = device_preprocess(v, form, t), fn(v, t)
        assert torch.equal(got, want), float((got - want).abs().max())


@pytest.mark.parametrize("hw", [(64, 64), (97, 131), (320, 240)])
def test_u8_equals_f32_of_bytes(hw):
    b = u8((2, 10) + hw + (3,), 7)
    f = b.float().permute(0, 1, 4, 2, 3).contiguous() / 255.
    from_u8 = device_preprocess(b, fvd.FORM_U8, 10)
    assert torch.equal(from_u8, device_preprocess(f, fvd.FORM_F32, 10))
    assert torch.equal(from_u8, device_preprocess(f, fvd.FORM_F32_TRUNC, 10))
    assert torch.equal(from_u8, so.preprocess_styleganv(f, 10))


def test_seeded_features_match_reference(golden, sgv):
    for name, case in golden["feats"].items():
        v = rand(case["shape"], case["seed"])
        got = sgv.features(fvd.SuiteClips(v.to(DEV), fvd.FORM_F32), case["shape"][1]).cpu()
        ref = case["feats"]
        err = float((got - ref).abs().max() / ref.abs().max())
        print(f"{name}: {err:.2e} of max|feature|")
        assert err <= 1e-4


@pytest.mark.skipif(not os.path.isfile(SHIPPED), reason="oracle/_ref/i3d_styleganv.pt not built")
def test_shipped_features_match_reference(golden):
    net = fvd.load_i3d_styleganv(DEV, SHIPPED)
    case = golden["shipped"]
    v = rand(case["shape"], case["seed"])
    got = net.features(fvd.SuiteClips(v.to(DEV), fvd.FORM_F32), case["shape"][1]).cpu()
    err = float((got - case["feats"]).abs().max() / case["feats"].abs().max())
    print(f"shipped weights: {err:.2e} of max|feature|")
    assert err <= 1e-4


def fvd_sets(golden):
    B, T, H, W = golden["fvd"]["set"]
    gt = u8((B, T, H, W, 3), golden["fvd"]["seed"])
    gen = gt.clone()
    gen[..., 1:, :] = gen[..., :-1, :]
    return gt, (gen.int() * 7 // 8 + 16).to(torch.uint8)


@pytest.mark.parametrize("method", ["styleganv", "videogpt"])
@pytest.mark.parametrize("inputs", ["u8_device", "f32_host"])
def test_calculate_fvd_matches_reference(golden, sgv, vgpt, method, inputs):
    gt, gen = fvd_sets(golden)
    if inputs == "u8_device":
        a, b = gt.to(DEV), gen.to(DEV)
    else:
        a, b = (x.float().permute(0, 1, 4, 2, 3).contiguous() / 255. for x in (gt, gen))
    r = quality.calculate_fvd(a, b, "cuda", method, i3d=sgv if method == "styleganv" else vgpt)
    ref = golden["fvd"][method]
    assert tuple(r["video_setting"]) == ref["video_setting"] and r["video_setting_name"] == ref["video_setting_name"]
    assert sorted(r["value"]) == sorted(ref["value"])
    for t, v in ref["value"].items():
        print(f"{method} t={t}: {r['value'][t]:.6f} reference {v:.6f} relative {abs(r['value'][t] / v - 1):.2e}")
        assert abs(r["value"][t] / v - 1) <= 1e-4


def test_prefix_workspace_equals_copied_prefix(sgv):
    v = u8((3, 14, 72, 88, 3), 11).to(DEV)
    full = fvd.SuiteClips(v, fvd.FORM_U8)
    for t in (10, 13):
        a = sgv.features(full, t).clone()
        b = sgv.features(fvd.SuiteClips(v[:, :t].contiguous(), fvd.FORM_U8), t)
        assert torch.equal(a, b)


def test_chunks_equal_single_clips(sgv):
    v = u8((23, 12, 48, 56, 3), 12).to(DEV)
    together = sgv.features(fvd.SuiteClips(v, fvd.FORM_U8), 12).clone()
    assert fvd.SUITE_CHUNK_FRAMES // 12 < 23                  # more than one chunk, and a ragged last one
    for i in (0, 5, 21, 22):
        alone = sgv.features(fvd.SuiteClips(v[i:i + 1].contiguous(), fvd.FORM_U8), 12)
        assert torch.equal(together[i:i + 1], alone), i


def test_graph_replay_equals_eager(sgv):
    c = fvd.SuiteClips(u8((2, 10, 64, 64, 3), 13).to(DEV), fvd.FORM_U8)
    sgv._suite_ws.pop((2, 10), None)
    outs = [sgv.features(c, 10).clone() for _ in range(3)]   # eager, capture + replay, replay
    assert isinstance(sgv._suite_ws[(2, 10)].graphs["i3d"], tuple)
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


def test_refusals_launch_nothing(sgv, vgpt):
    a = torch.zeros(2, 12, 64, 64, 3, dtype=torch.uint8, device=DEV)
    n0 = _cabi.launch_count
    for args, kw in [((a, a[:, :11]), {"i3d": sgv}), ((a, a), {"i3d": vgpt}), ((a, a.float()), {"i3d": sgv}),
                     ((a, a), {"i3d": sgv, "method": "fid"})]:
        with pytest.raises((TypeError, ValueError)):
            quality.calculate_fvd(*args, "cuda", **kw)
    with pytest.raises(ValueError):
        sgv.logits(a)
    assert _cabi.launch_count == n0


def test_fvd_external_selects_frames(vgpt):
    gt = [u8((n, 64, 64, 3), 20 + n) for n in (17, 20, 25)]
    gen = [u8((n, 64, 64, 3), 40 + n) for n in (18, 17, 30)]
    r = consumers.fvd_external(gt, gen, vgpt, frames=11, sampling="center")
    sel = lambda clips: torch.stack([c[list(consumers.fvd_external_indices(len(c), 11))] for c in clips]).to(DEV)
    ref = quality.calculate_fvd(sel(gt), sel(gen), "cuda", "videogpt", i3d=vgpt)
    assert r == ref and sorted(r["value"]) == [10, 11]
