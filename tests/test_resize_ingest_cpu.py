"""CPU checks of the image-resize input side: the host coefficient tables (layout.resample_coeffs) with the tap-by-tap integer
arithmetic of omt_resample_u8 (layout.resize_u8) equal Pillow's resize byte for byte, the parameter helper consumes torch's
CPU generator as torchvision's RandomCrop / RandomHorizontalFlip do, and the golden fixture is reproduced."""
import numpy as np
import pytest
import torch

from omnitokenizer_b200 import layout as L
from oracle import make_golden_resize as G
from tests.util import load_golden

PRESETS = {"image": L.image_resize, "resizecrop": L.resizecrop_resize, "dit": L.dit_resize}

# (H, W) -> (h, w): down- and upscales from 1 x 1 to 4 000-pixel sides, ratios of 1 : 60 both ways, identity axes, and
# images taller than 100x their width (Pillow's vertical-first order)
SWEEP = [((375, 500), (256, 256)), ((333, 500), (256, 341)), ((100, 80), (256, 256)), ((17, 1000), (384, 384)),
         ((1, 1), (7, 5)), ((1, 1), (1, 1)), ((5, 7), (1, 1)), ((1, 60), (60, 1)), ((60, 1), (1, 60)), ((600, 10), (10, 600)),
         ((3, 4000), (5, 64)), ((4000, 2), (67, 3)), ((4000, 2), (67, 2)), ((4001, 40), (10, 3)), ((2, 4100), (2, 4100)),
         ((3000, 4000), (256, 256)), ((31, 17), (256, 256)), ((64, 64), (64, 64)), ((64, 64), (64, 32)),
         ((48, 64), (48, 60)), ((256, 256), (384, 384)), ((16, 16), (960, 17))]


def _pillow(img: torch.Tensor, size, filt):
    from PIL import Image
    f = {"bicubic": Image.BICUBIC, "bilinear": Image.BILINEAR, "box": Image.BOX}[filt]
    return torch.from_numpy(np.asarray(Image.fromarray(img.numpy()).resize((size[1], size[0]), f)).copy())


@pytest.mark.parametrize("filt", ["bicubic", "bilinear", "box"])
def test_host_resize_equals_pillow(filt):
    pytest.importorskip("PIL")
    g = torch.Generator().manual_seed(3)
    for src, dst in SWEEP:
        if filt == "box" and max(src) > 1000:
            continue
        img = torch.randint(0, 256, src + (3,), generator=g, dtype=torch.uint8)
        got = L.resize_u8(img, L.U8Resize(dst, filt))
        assert torch.equal(got, _pillow(img, dst, filt)), f"{src} -> {dst} {filt}"


def test_coeffs_are_normalised_fixed_point():
    for n_in, n_out in ((500, 256), (256, 500), (1, 256), (4000, 67), (60, 1)):
        for filt in ("bicubic", "bilinear", "box"):
            bounds, k = L.resample_coeffs(n_in, n_out, filt)
            assert bounds.dtype == np.int32 and k.dtype == np.int32 and bounds.shape == (n_out, 2)
            assert (bounds[:, 0] >= 0).all() and (bounds.sum(1) <= n_in).all() and (bounds[:, 1] <= k.shape[1]).all()
            for i in range(n_out):
                assert not k[i, bounds[i, 1]:].any()
                assert abs(int(k[i].sum()) - (1 << 22)) <= k.shape[1]
    assert L.resample_coeffs(500, 256, "bicubic") is L.resample_coeffs(500, 256, "bicubic")      # cached per key


@pytest.mark.parametrize("name", list(PRESETS))
def test_presets_through_torchvision(name):
    """The presets composed as the loaders compose them, with their random draws: the helper's parameters and the host
    resize reproduce torchvision + Pillow's bytes, and leave the CPU generator where the transforms leave it."""
    pytest.importorskip("PIL")
    pytest.importorskip("torchvision")
    from PIL import Image
    res = 24
    tf, drawn = G.transforms_by_name(res)[name]
    rz = PRESETS[name](res)
    g = torch.Generator().manual_seed(4)
    imgs = [torch.randint(0, 256, (int(h), int(w), 3), generator=g, dtype=torch.uint8)
            for h, w in torch.randint(1, 90, (12, 2), generator=g).tolist()] + [torch.zeros(36, 36, 3, dtype=torch.uint8)]
    torch.manual_seed(123)
    want, want_params = [], []
    for im in imgs:
        want.append(torch.from_numpy(np.asarray(tf(Image.fromarray(im.numpy()))).copy()))
        want_params.append(drawn())
    rng = torch.get_rng_state()
    torch.manual_seed(123)
    params = L.resize_params(len(imgs), rz)
    assert params == want_params
    assert torch.equal(torch.get_rng_state(), rng)
    for im, p, w in zip(imgs, params, want):
        assert torch.equal(L.resize_u8(im, rz, p), w)
    if name == "resizecrop":
        assert len({p[:2] for p in params}) > 1
    if name == "dit":
        assert {p[2] for p in params} == {False, True}


def test_resize_params_draw_nothing_without_randomness():
    torch.manual_seed(0)
    st = torch.get_rng_state()
    assert L.resize_params(5, L.image_resize(32)) == [(0, 0, False)] * 5
    assert L.resize_params(3, L.U8Resize((32, 32), crop=32)) == [(0, 0, False)] * 3     # RandomCrop of the whole image
    assert torch.equal(torch.get_rng_state(), st)


def test_golden_fixture_reproduced():
    pytest.importorskip("PIL")
    pytest.importorskip("torchvision")
    want = load_golden("u8_resize")
    got = G.build(want["res"], want["seed"])
    assert got["sizes"] == want["sizes"] and got["source_sum"] == want["source_sum"]
    for name in PRESETS:
        assert torch.equal(got[name]["out"], want[name]["out"]) and got[name]["params"] == want[name]["params"]
        assert torch.equal(got[name]["rng_after"], want[name]["rng_after"])


@pytest.mark.parametrize("name", list(PRESETS))
def test_host_resize_equals_golden(name):
    """No Pillow needed: the fixture's sources, parameters and bytes against layout.resize_u8 / resize_params."""
    fx = load_golden("u8_resize")
    srcs = G.sources(fx["source_seed"])
    assert [int(s.long().sum()) for s in srcs] == fx["source_sum"]
    rz = PRESETS[name](fx["res"])
    torch.manual_seed(fx["seed"])
    assert L.resize_params(len(srcs), rz) == fx[name]["params"]
    assert torch.equal(torch.get_rng_state(), fx[name]["rng_after"])
    got = torch.stack([L.resize_u8(s, rz, p) for s, p in zip(srcs, fx[name]["params"])])
    assert torch.equal(got, fx[name]["out"])


def test_resize_spec_checks():
    with pytest.raises(ValueError, match="crop"):
        L.check_resize(L.U8Resize((32, 32), crop=40))
    with pytest.raises(ValueError, match="filter"):
        L.check_resize(L.U8Resize((32, 32), "lanczos"))
    with pytest.raises(TypeError):
        L.check_resize((32, 32))
    rz = L.resizecrop_resize(32)
    assert rz.size == (48, 48) and rz.out_size == (32, 32)
    with pytest.raises(ValueError, match="not a draw"):
        L.check_resize_params([(17, 0, False)], 1, rz)
    with pytest.raises(ValueError, match="not a draw"):
        L.check_resize_params([(0, 0, True)], 1, rz)
    with pytest.raises(ValueError, match="2 resize parameters for 1"):
        L.check_resize_params([(0, 0, False)] * 2, 1, rz)


def test_consumers_transform_on_the_host_for_other_models():
    """A model without encode_images_u8 gets the host-transformed stack through its uint8 (or fp32) path, with the
    transform's parameters drawn first, as the loader draws them."""
    from omnitokenizer_b200 import consumers as C

    class Fake:
        def __init__(self):
            self.seen = []

        def encode_u8(self, frames, is_image, include_embeddings=False, norm=None):
            self.seen.append((frames.clone(), is_image, norm))
            return torch.ones(frames.shape[0], 8, 1, 2, 2)

    g = torch.Generator().manual_seed(9)
    imgs = [torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8) for h, w in ((50, 70), (9, 9), (32, 32))]
    fake = Fake()
    torch.manual_seed(2)
    z = C.dit_encode_latents_images_u8(fake, imgs, 32)
    torch.manual_seed(2)
    params = L.resize_params(3, L.dit_resize(32))
    want = torch.stack([L.resize_u8(im, L.dit_resize(32), p) for im, p in zip(imgs, params)])
    frames, is_image, norm = fake.seen[0]
    assert torch.equal(frames, want) and is_image and norm == C.IMAGE_NORM
    assert torch.equal(z, torch.full((3, 8, 1, 2, 2), C.LATENT_SCALE))
