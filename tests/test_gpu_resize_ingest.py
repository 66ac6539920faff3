"""GPU checks of the image-resize input side: omt_resample_u8 against the golden fixture (torchvision + Pillow) and live
Pillow on ragged batches, per-image isolation, and encode_images_u8 / forward_images_u8 against encode_u8 / forward_u8 on
the host-transformed images.  Every comparison is exact (torch.equal)."""
import numpy as np
import pytest
import torch

from omnitokenizer_b200 import _cabi
from omnitokenizer_b200 import consumers as C
from omnitokenizer_b200 import layout as L
from oracle import make_golden_resize as G
from oracle import omni_oracle as oo
from oracle import weights as W
from tests.util import build_model, load_golden

pytestmark = pytest.mark.gpu
PRESETS = {"image": L.image_resize, "resizecrop": L.resizecrop_resize, "dit": L.dit_resize}


def _img(h, w, seed):
    return torch.randint(0, 256, (h, w, 3), generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)


def _want(images, rz, params):
    """Pillow + the crop / flip when Pillow imports, else the host twin (itself pinned to Pillow by the CPU tests)."""
    try:
        from PIL import Image
    except ImportError:
        return torch.stack([L.resize_u8(im, rz, p) for im, p in zip(images, params)])
    f = {"bicubic": Image.BICUBIC, "bilinear": Image.BILINEAR, "box": Image.BOX}[rz.filter]
    (h, w), (oh, ow) = rz.size, rz.out_size
    outs = []
    for im, (i, j, flip) in zip(images, params):
        o = torch.from_numpy(np.asarray(Image.fromarray(im.numpy()).resize((w, h), f)).copy())[i:i + oh, j:j + ow]
        outs.append(o.flip(1) if flip else o)
    return torch.stack(outs)


@pytest.fixture(scope="module")
def model(cuda):
    cfg = oo.Config(resolution=64)
    return build_model(cfg, W.make_state_dict(cfg, 3), cuda, "f16x3")


def _resample(m, images, rz, params):
    oh, ow = rz.out_size
    out = torch.full((len(images), 1, oh, ow, 3), 7, dtype=torch.uint8, device=m.device)
    m.engine().resample_u8(images, rz, params, out)
    return out[:, 0].cpu()


@pytest.mark.parametrize("name", list(PRESETS))
def test_resample_equals_golden(model, name):
    fx = load_golden("u8_resize")
    srcs = G.sources(fx["source_seed"])
    rz = PRESETS[name](fx["res"])
    assert torch.equal(_resample(model, srcs, rz, fx[name]["params"]), fx[name]["out"])


def test_resample_ragged_batch_equals_pillow(model):
    """Photo-sized, 4000 x 3000, 31 x 17 upscale, extreme aspect, 1-pixel, at-size and vertical-first images in one batch,
    through each preset at 256 (and 384 / 256 crop), then each image alone: the same bytes (no neighbour leaks in)."""
    sizes = [(375, 500), (3000, 4000), (31, 17), (1, 1), (2, 900), (900, 2), (256, 256), (384, 384), (60, 1), (1, 60),
             (333, 500), (500, 333), (8000, 40), (17, 1000)]
    imgs = [_img(h, w, 100 + k) for k, (h, w) in enumerate(sizes)]
    for name, preset in PRESETS.items():
        rz = preset(256)
        torch.manual_seed(5)
        params = L.resize_params(len(imgs), rz)
        got = _resample(model, imgs, rz, params)
        assert torch.equal(got, _want(imgs, rz, params)), name
        for k in (0, 2, 3, 12):
            assert torch.equal(_resample(model, [imgs[k]], rz, [params[k]])[0], got[k]), (name, sizes[k])


def _usage(m):
    return m.codebook.codebook_usage.clone(), m.codebook.call_cnt


def _set_usage(m, st):
    m.codebook.codebook_usage.data = st[0].clone()
    m.codebook.call_cnt = st[1]


def _eq(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_eq(a[k], b[k]) for k in a)
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(_eq(x, y) for x, y in zip(a, b))
    if a is None or b is None:
        return a is b
    return torch.equal(a, b)


def _host_stack(images, rz):
    params = L.resize_params(len(images), rz)
    return torch.stack([L.resize_u8(im, rz, p) for im, p in zip(images, params)])


@pytest.mark.parametrize("math", ["f16x3", "f16x1"])
@pytest.mark.parametrize("vae", [False, True])
def test_encode_and_forward_images_u8_equal_u8_path(cuda, math, vae):
    cfg = oo.Config(resolution=64, use_vae=vae)
    m = build_model(cfg, W.make_state_dict(cfg, 4), cuda, math)
    imgs = [_img(h, w, 200 + k) for k, (h, w) in enumerate([(375, 500), (31, 17), (64, 64), (96, 120), (1, 3), (700, 5)])]
    st0 = _usage(m)
    for rz in (L.image_resize(64), L.resizecrop_resize(64), L.dit_resize(64)):
        for emb in ((False, True) if not vae else (False,)):
            for _ in range(3):                   # eager, graph capture, graph replay of the shared encode_u8 graph
                _set_usage(m, st0)
                torch.manual_seed(11)
                want = m.encode_u8(_host_stack(imgs, rz).to(cuda), True, include_embeddings=emb, norm=C.IMAGE_NORM)
                st_want, rng_want = _usage(m), torch.get_rng_state()
                _set_usage(m, st0)
                torch.manual_seed(11)
                got = m.encode_images_u8(imgs, rz, include_embeddings=emb)
                assert _eq(got, want), (rz, emb)
                assert _eq(_usage(m)[0], st_want[0]) and _usage(m)[1] == st_want[1]
                assert torch.equal(torch.get_rng_state(), rng_want)
        _set_usage(m, st0)
        torch.manual_seed(12)
        want = m.forward_u8(_host_stack(imgs, rz).to(cuda), C.IMAGE_NORM)
        st_want, rng_want = _usage(m), torch.get_rng_state()
        _set_usage(m, st0)
        torch.manual_seed(12)
        got = m.forward_images_u8(imgs, rz)
        assert _eq(got, want)
        assert _eq(_usage(m)[0], st_want[0]) and _usage(m)[1] == st_want[1]
        assert torch.equal(torch.get_rng_state(), rng_want)
    # the consumers over the same images
    torch.manual_seed(13)
    if vae:
        want = m.encode_u8(_host_stack(imgs, L.dit_resize(64)).to(cuda), True, norm=C.IMAGE_NORM).mul_(C.LATENT_SCALE)
        torch.manual_seed(13)
        assert torch.equal(C.dit_encode_latents_images_u8(m, imgs, 64), want)
    else:
        want = C.encode_to_z_u8(m, _host_stack(imgs, L.image_resize(64)).to(cuda), True, norm=C.IMAGE_NORM)
        torch.manual_seed(13)
        assert _eq(C.encode_to_z_images_u8(m, imgs, L.image_resize(64)), want)


def test_second_batch_of_other_sizes_reuses_encode_u8_slot_graph(model, cuda):
    """Batches of different source sizes at the same output shape share encode_u8's graph of that shape and stay exact."""
    rz = L.image_resize(64)
    batches = [[_img(h, w, 300 + 10 * b + k) for k, (h, w) in enumerate(sz)]
               for b, sz in enumerate([[(375, 500), (80, 90)], [(17, 23), (640, 480)], [(64, 64), (1, 1)], [(200, 2), (3, 3000)]])]
    graphs = []
    for imgs in batches:
        want = model.encode_u8(_host_stack(imgs, rz).to(cuda), True, norm=C.IMAGE_NORM)
        assert torch.equal(model.encode_images_u8(imgs, rz), want)
        ws = model.engine()._workspace(2 * 8 * 8)                # 2 images on the 8 x 8 token grid
        graphs.append(ws.graphs_of("encode_u8"))
    assert len(graphs[-1]) == 1
    g = next(iter(graphs[-1].values()))
    assert not isinstance(g, str) and next(iter(graphs[2].values())) is g


def test_malformed_input_raises_before_launch(model, cuda):
    m = model
    rz = L.image_resize(64)
    ok = _img(40, 50, 1)
    n0 = _cabi.launch_count
    with pytest.raises(TypeError):
        m.encode_images_u8([ok.float()], rz)
    with pytest.raises(ValueError, match=r"\(H, W, 3\)"):
        m.encode_images_u8([ok[..., :2].contiguous()], rz)
    with pytest.raises(ValueError, match=r"\(H, W, 3\)"):
        m.encode_images_u8([torch.zeros(0, 5, 3, dtype=torch.uint8)], rz)
    with pytest.raises(ValueError, match="host memory"):
        m.encode_images_u8([ok.to(cuda)], rz)
    with pytest.raises(ValueError, match="square with side a multiple of the patch size"):
        m.encode_images_u8([ok], L.image_resize(60))
    with pytest.raises(ValueError, match="not a draw"):
        m.encode_images_u8([ok], L.resizecrop_resize(64), params=[(40, 0, False)])
    with pytest.raises(ValueError, match="needs at least one image"):
        m.forward_images_u8([], rz)
    assert _cabi.launch_count == n0
    # an empty list is encode_u8's B = 0 result
    e = m.encode_images_u8([], rz)
    assert tuple(e.shape) == (0, 1, 8, 8) and e.dtype == torch.int64
    # the entry point checks descriptors against the buffers before its launch
    eng = m.engine()
    args = list(eng.stage_images_u8([ok, _img(9, 9, 2)], rz, [(0, 0, False)] * 2))
    torch.cuda.synchronize()
    out = torch.empty(2, 64, 64, 3, dtype=torch.uint8, device=cuda)
    host = eng._stage
    desc = host[:2 * 72].view(torch.int32).view(2, 18)       # int64 source offset, then H, W, rh, rw, y0, x0, flip, ...
    tab = host[144:148].view(torch.int32)                     # xmin of the first output column of the first table
    for t, field, value, msg in ((desc[1], 2, 0, "source 0x9"), (desc[1], 6, 1, "crop"), (desc[1], 7, -1, "crop"),
                                 (desc[1], 11, 1 << 20, "horizontal table"), (desc[1], 9, 0, "no horizontal pass"),
                                 (desc[1], 17, 2, "v_first"), (tab, 0, 1000, "taps outside the source")):
        saved = int(t[field])
        t[field] = value
        with pytest.raises(RuntimeError, match=msg):
            _cabi.call("omt_resample_u8", *args, out)
        t[field] = saved
    bad = list(args)
    bad[1] = args[1] - 1                         # one source byte short
    with pytest.raises(RuntimeError, match="outside the"):
        _cabi.call("omt_resample_u8", *bad, out)
    bad = list(args)
    bad[0] = None
    with pytest.raises(RuntimeError, match="null"):
        _cabi.call("omt_resample_u8", *bad, out)
    bad = list(args)
    bad[8] = 0
    with pytest.raises(RuntimeError, match="output 0x64"):
        _cabi.call("omt_resample_u8", *bad, out)
    # the tables restored, the same arguments run
    _cabi.call("omt_resample_u8", *args, out)
    assert torch.equal(out.cpu(), _want([ok, _img(9, 9, 2)], rz, [(0, 0, False)] * 2))
