"""GPU checks of the video-clip input side: omt_resample_clips against the golden fixture (the reference's video
transforms) and the host twin, and encode_clips_u8 / latte_encode_latents_clips_u8 against encode / latte_encode_latents
of the host pipeline.  Every comparison is exact; floats are compared as int32 bit patterns."""
import random

import pytest
import torch

from omnitokenizer_b200 import _cabi
from omnitokenizer_b200 import consumers as C
from omnitokenizer_b200 import layout as L
from oracle import make_golden_clips as G
from oracle import omni_oracle as oo
from oracle import weights as W
from tests.util import build_model, load_golden

pytestmark = pytest.mark.gpu
PRESETS = {"ucf": L.ucf_clip_resize, "sky": L.sky_clip_resize, "taichi": lambda s: L.taichi_clip_resize()}


def _bits(t):
    return t.contiguous().view(torch.int32)


def _clip(F, h, w, seed):
    return torch.randint(0, 256, (F, h, w, 3), generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)


@pytest.fixture(scope="module")
def model(cuda):
    cfg = oo.Config(resolution=64)
    return build_model(cfg, W.make_state_dict(cfg, 3), cuda, "f16x3")


def _resample(m, clips, rz, flips, norm=C.LATTE_NORM):
    F, H, W_ = clips[0].shape[:3]
    oh, ow = L.clip_out_size(H, W_, rz)
    out = torch.full((len(clips), 3, F, oh, ow), float("nan"), device=m.device)    # an unwritten element shows
    m.engine().resample_clips(clips, rz, flips, norm, out)
    return out.cpu()


def _host(clips, rz, flips, norm=C.LATTE_NORM):
    return torch.stack([L.resize_clip(c, rz, f, norm).transpose(0, 1) for c, f in zip(clips, flips)])   # (B, 3, F, h, w)


@pytest.mark.parametrize("name", list(PRESETS))
def test_kernel_equals_golden(model, name):
    fx = load_golden("clip_resize")
    srcs = G.sources(fx["taichi_sizes"] if name == "taichi" else fx["sizes"], fx["source_seed"], fx["frames"])
    rz = PRESETS[name](fx["s"])
    flips = fx[name]["flips"]
    if name == "taichi":           # no resize: each clip keeps its own size, so each is its own batch
        for c, f, want in zip(srcs, flips, fx[name]["out"]):
            assert torch.equal(_bits(_resample(model, [c], rz, [f])[0]), _bits(want.transpose(0, 1)))
        return
    got = _resample(model, srcs, rz, flips)
    want = torch.stack([o.transpose(0, 1) for o in fx[name]["out"]])
    assert torch.equal(_bits(got), _bits(want))


def test_kernel_equals_host_twin_sweep(model):
    """All three presets (both of torch's arithmetic forms), flip on and off, F in {1, 5, 17}, a ragged batch."""
    sizes = [(240, 320), (320, 240), (1, 1), (2, 3), (37, 1000), (250, 333), (64, 64), (45, 64)]
    for F in (1, 5, 17):
        clips = [_clip(F, h, w, 10 * F + k) for k, (h, w) in enumerate(sizes)]
        flips = [k % 2 == 1 for k in range(len(sizes))]
        for rz in (L.ucf_clip_resize(64), L.ClipResize("scale_crop", 128, True, in_workers=False), L.sky_clip_resize(64),
                   L.ClipResize("crop_resize", 96, False, in_workers=False)):
            got = _resample(model, clips, rz, flips)
            assert torch.equal(_bits(got), _bits(_host(clips, rz, flips))), (F, rz)
            assert torch.equal(_bits(_resample(model, [clips[3]], rz, [flips[3]])[0]), _bits(got[3]))
        tz = [_clip(F, 24, 40, 500 + k) for k in range(3)]
        tf = [True, False, True]
        assert torch.equal(_bits(_resample(model, tz, L.taichi_clip_resize(), tf)), _bits(_host(tz, L.taichi_clip_resize(), tf)))


def _usage(m):
    return m.codebook.codebook_usage.clone(), m.codebook.call_cnt


def _set_usage(m, st):
    m.codebook.codebook_usage.data = st[0].clone()
    m.codebook.call_cnt = st[1]


def _eq(a, b):
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(_eq(x, y) for x, y in zip(a, b))
    return torch.equal(_bits(a) if a.is_floating_point() else a, _bits(b) if b.is_floating_point() else b)


def _host_stack(clips, rz):
    """The loader's pipeline on the host with its own flip draws: (B, 3, F, h, w) fp32, 'b f c h w -> b c f h w'."""
    flips = L.clip_params(len(clips), rz)
    return _host(clips, rz, flips)


@pytest.mark.parametrize("math", ["f16x3", "fp32", "f16x1"])
@pytest.mark.parametrize("vae", [False, True])
def test_encode_clips_u8_equals_encode_of_host_pipeline(cuda, math, vae):
    cfg = oo.Config(resolution=64, use_vae=vae)
    m = build_model(cfg, W.make_state_dict(cfg, 4), cuda, math)
    clips = [_clip(5, h, w, 200 + k) for k, (h, w) in enumerate([(240, 320), (31, 17), (64, 64), (96, 120), (1, 3)])]
    st0 = _usage(m)
    for rz in (L.ucf_clip_resize(64), L.sky_clip_resize(64)):
        for emb in ((False, True) if not vae else (False,)):
            for _ in range(3):                   # eager, graph capture, graph replay of encode's graph of the shape
                _set_usage(m, st0)
                random.seed(7)
                torch.manual_seed(11)
                want = m.encode(_host_stack(clips, rz).to(cuda), False, include_embeddings=emb)
                st_want, rng_want, py_want = _usage(m), torch.get_rng_state(), random.getstate()
                _set_usage(m, st0)
                random.seed(7)
                torch.manual_seed(11)
                got = m.encode_clips_u8(clips, rz, include_embeddings=emb)
                assert _eq(got, want), (rz, emb)
                assert _eq(_usage(m)[0], st_want[0]) and _usage(m)[1] == st_want[1]
                assert torch.equal(torch.get_rng_state(), rng_want) and random.getstate() == py_want
    if not vae:                                  # Latte's consumer takes VAE latents
        return
    random.seed(8)
    torch.manual_seed(13)
    want = C.latte_encode_latents(m, _host_stack(clips, L.ucf_clip_resize(64)).transpose(1, 2).to(cuda))
    rng_want, py_want = torch.get_rng_state(), random.getstate()
    random.seed(8)
    torch.manual_seed(13)
    got = C.latte_encode_latents_clips_u8(m, clips, L.ucf_clip_resize(64))
    assert _eq(got, want) and torch.equal(torch.get_rng_state(), rng_want) and random.getstate() == py_want


def test_ucf_config_full_size(cuda):
    """Latte's ucf101 config: 5 clips of 17 x 240 x 320 at 256^2, VAE latents of the consumer."""
    cfg = oo.Config(resolution=256, use_vae=True)
    m = build_model(cfg, W.make_state_dict(cfg, 5), cuda, "f16x3")
    clips = [_clip(17, 240, 320, 900 + k) for k in range(5)]
    rz = L.ucf_clip_resize(256)
    random.seed(3)
    got_x = _resample(m, clips, rz, L.clip_params(5, rz))
    random.seed(3)
    assert torch.equal(_bits(got_x), _bits(_host_stack(clips, rz)))
    random.seed(4)
    torch.manual_seed(5)
    want = C.latte_encode_latents(m, _host_stack(clips, rz).transpose(1, 2).to(cuda))
    random.seed(4)
    torch.manual_seed(5)
    got = C.latte_encode_latents_clips_u8(m, clips, rz)
    assert got.shape[:2] == (5, 5) and _eq(got, want)


def test_second_batch_of_other_sizes_reuses_encode_slot_graph(model, cuda):
    rz = L.ucf_clip_resize(64)
    batches = [[_clip(5, h, w, 300 + 10 * b + k) for k, (h, w) in enumerate(sz)]
               for b, sz in enumerate([[(240, 320), (80, 90)], [(17, 23), (640, 480)], [(64, 64), (1, 1)], [(200, 70), (3, 300)]])]
    graphs = []
    for clips in batches:
        random.seed(1)
        want = model.encode(_host_stack(clips, rz).to(cuda), False)
        random.seed(1)
        assert torch.equal(model.encode_clips_u8(clips, rz), want)
        ws = model.engine()._workspace(2 * 2 * 8 * 8)            # 2 clips of T' = 2 on the 8 x 8 token grid
        graphs.append(ws.graphs_of("encode"))
    assert len(graphs[-1]) == 1
    g = next(iter(graphs[-1].values()))
    assert not isinstance(g, str) and next(iter(graphs[2].values())) is g


def test_malformed_input_raises_before_launch(model, cuda):
    m = model
    rz = L.ucf_clip_resize(64)
    ok = _clip(5, 40, 50, 1)
    n0 = _cabi.launch_count
    with pytest.raises(ValueError, match="no smaller than crop_size"):
        m.encode_clips_u8([ok, _clip(5, 239, 300, 2)], L.ucf_clip_resize(256))
    with pytest.raises(ValueError, match="same number of frames"):
        m.encode_clips_u8([ok, _clip(9, 40, 50, 2)], rz)
    with pytest.raises(AssertionError, match="divisible by temporal patch size"):
        m.encode_clips_u8([_clip(16, 40, 50, 2)], rz)
    with pytest.raises(ValueError, match=r"\(F, H, W, 3\)"):
        m.encode_clips_u8([torch.zeros(5, 40, 50, 4, dtype=torch.uint8)], rz)
    with pytest.raises(ValueError, match="host memory"):
        m.encode_clips_u8([ok.to(cuda)], rz)
    with pytest.raises(TypeError):
        m.encode_clips_u8([ok.float()], rz)
    with pytest.raises(ValueError, match="not a draw"):
        m.encode_clips_u8([ok], L.sky_clip_resize(64), params=[True])
    with pytest.raises(ValueError, match="largest byte"):
        m.encode_clips_u8([ok], rz, norm=C.VIDEO_NORM)
    with pytest.raises(ValueError, match="square with side a multiple of the patch size"):
        m.encode_clips_u8([ok], L.ucf_clip_resize(60))
    assert _cabi.launch_count == n0
    # the entry point checks descriptors against the buffers before its launch
    eng = m.engine()
    clips = [ok, _clip(5, 9, 9, 2)]
    args, (B, F, oh, ow) = eng.stage_clips_u8(clips, rz, [False, True])
    torch.cuda.synchronize()
    lut = eng._table(("clipnorm", C.LATTE_NORM), lambda: L.clip_norm_table(C.LATTE_NORM))
    out = torch.empty(B, 3, F, oh, ow, device=cuda)
    desc = eng._stage[:2 * 64].view(torch.int32).view(2, 16)   # int64 source offset, then H, W, y0, x0, wh, ww, rh, ...
    tab = eng._stage[args[4] - args[2]:][:16].view(torch.int32)  # first entry of the first table
    for t, field, value, msg in ((desc[1], 2, 10, "outside the"), (desc[1], 4, 1, "window"), (desc[1], 10, 9, "crop"),
                                 (desc[1], 12, 2, "flip / form"), (desc[1], 13, 1 << 20, "vertical table"),
                                 (desc[1], 14, 2, "horizontal table"), (tab, 1, 1000, "indices outside")):
        saved = int(t[field])
        t[field] = value
        with pytest.raises(RuntimeError, match=msg):
            _cabi.call("omt_resample_clips", *args, lut, B, F, oh, ow, out)
        t[field] = saved
    bad = list(args)
    bad[1] = args[1] - 1
    with pytest.raises(RuntimeError, match="outside the"):
        _cabi.call("omt_resample_clips", *bad, lut, B, F, oh, ow, out)
    with pytest.raises(RuntimeError, match="null"):
        _cabi.call("omt_resample_clips", *args, None, B, F, oh, ow, out)
    _cabi.call("omt_resample_clips", *args, lut, B, F, oh, ow, out)
    assert torch.equal(_bits(out.cpu()), _bits(_host(clips, rz, [False, True])))
