"""omt_jpeg_roundtrip_u8 on the device: Pillow's JPEG save and reload byte for byte on the seeded grid of
oracle/jpeg_oracle.py, one image at a time and in batches, against Pillow run live and tests/golden/jpeg_roundtrip.pt;
no write outside the output, src untouched, identical bytes on a second launch, refusals with no launch and no write;
and eval_step_fid(saved_as="jpeg") against the script's bytes saved and reopened by Pillow."""
import ctypes
import io

import numpy as np
import pytest
import torch

from oracle import jpeg_oracle as J
from oracle.make_golden_jpeg import pillow_roundtrip, sha
from omnitokenizer_b200 import _cabi, consumers as C, fid, jpeg
from omnitokenizer_b200 import layout as L
from tests.util import load_golden

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SENTINEL = 0xA5
GUARD = 4096


@pytest.fixture(scope="module")
def golden():
    return load_golden("jpeg_roundtrip")


def _dev(x: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def test_kernel_equals_pillow_and_golden(golden):
    bad = []
    for c in golden["cases"]:
        x = J.content(c["kind"], c["H"], c["W"], c["seed"])
        got = jpeg.roundtrip_u8(_dev(x)[None], c["quality"])[0].cpu().numpy()
        want, _ = pillow_roundtrip(x, c["quality"])
        if not (np.array_equal(got, want) and sha(got) == c["output_sha"]):
            bad.append((c["H"], c["W"], c["quality"], c["kind"], int((got != want).sum())))
        if "output" in c:
            assert np.array_equal(got, c["output"].numpy())
    assert not bad, f"{len(bad)} of {len(golden['cases'])} cases differ, first {bad[:5]}"


@pytest.mark.parametrize("B, H, W, q", [(5, 1, 1, 75), (4, 3, 5, 20), (3, 17, 18, 75), (6, 85, 85, 75),
                                        (2, 255, 257, 90), (64, 256, 256, 75), (50, 128, 128, 75), (3, 100, 33, 1)])
def test_batches_equal_pillow(B, H, W, q):
    xs = [J.content(J.KINDS[i % len(J.KINDS)], H, W, 7000 + i) for i in range(B)]
    got = jpeg.roundtrip_u8(_dev(np.stack(xs)), q).cpu().numpy()
    for i, x in enumerate(xs):
        assert np.array_equal(got[i], pillow_roundtrip(x, q)[0]), (i, J.KINDS[i % len(J.KINDS)])


def _guarded(n: int, fill=SENTINEL):
    buf = torch.full((GUARD + n + GUARD,), fill, dtype=torch.uint8, device=DEV)
    return buf, buf[GUARD:GUARD + n]


@pytest.mark.parametrize("B, H, W", [(3, 85, 85), (2, 1, 3), (2, 33, 17)])
def test_no_write_outside_output_and_src_kept(B, H, W):
    xs = np.stack([J.content("noise", H, W, 50 + i) for i in range(B)])
    sbuf, src = _guarded(xs.size, 0x5A)
    src.copy_(torch.from_numpy(xs.reshape(-1)))
    src_before = sbuf.clone()
    dbuf, dst = _guarded(xs.size)
    nscr = jpeg.scratch_bytes(B, H, W)
    kbuf, scratch = _guarded(nscr)
    tables = np.ascontiguousarray(jpeg.quant_tables(75))
    outs = []
    for _ in range(2):
        _cabi.call("omt_jpeg_roundtrip_u8", src, dst, B, H, W, tables.ctypes.data, scratch)
        torch.cuda.synchronize()
        outs.append(dst.clone())
    assert torch.equal(sbuf, src_before)
    for buf in (dbuf, kbuf):
        assert bool((buf[:GUARD] == SENTINEL).all()) and bool((buf[-GUARD:] == SENTINEL).all())
    assert torch.equal(outs[0], outs[1])
    got = outs[0].view(B, H, W, 3).cpu().numpy()
    for i in range(B):
        assert np.array_equal(got[i], pillow_roundtrip(xs[i], 75)[0])


def test_two_calls_give_identical_bytes():
    x = _dev(np.stack([J.content(k, 256, 256, 90 + i) for i, k in enumerate(J.KINDS)]))
    a = jpeg.roundtrip_u8(x)
    b = jpeg.roundtrip_u8(x)
    assert torch.equal(a, b) and a.data_ptr() != b.data_ptr()


def _refused(args, match):
    before = _cabi.launch_count
    with pytest.raises(RuntimeError, match=match):
        _cabi.call("omt_jpeg_roundtrip_u8", *args)
    assert _cabi.launch_count == before


def test_refusals_launch_nothing_and_write_nothing():
    B, H, W = 2, 20, 24
    src = torch.randint(0, 256, (B, H, W, 3), dtype=torch.uint8, device=DEV)
    dst = torch.full_like(src, SENTINEL)
    scratch = torch.full((jpeg.scratch_bytes(B, H, W) + 8,), SENTINEL, dtype=torch.uint8, device=DEV)
    good = np.ascontiguousarray(jpeg.quant_tables(75))
    t = good.ctypes.data
    _refused((None, dst, B, H, W, t, scratch), "null pointer")
    _refused((src, None, B, H, W, t, scratch), "null pointer")
    _refused((src, dst, B, H, W, None, scratch), "null pointer")
    _refused((src, dst, B, H, W, t, None), "null pointer")
    _refused((src, dst, -1, H, W, t, scratch), "B=-1")
    _refused((src, dst, B, 0, W, t, scratch), "images of")
    _refused((src, dst, B, H, 0, t, scratch), "images of")
    for i, v in ((0, 0), (5, 256), (64, 0), (127, 1000)):
        bad = good.copy()
        bad.reshape(-1)[i] = v
        _refused((src, dst, B, H, W, bad.ctypes.data, scratch), "outside 1..255")
    _refused((src, dst, 1, 40000, 40000, t, scratch), "overflow int32")
    _refused((src, dst, B, H, W, t, scratch[1:]), "8-byte aligned")
    _refused((src, src, B, H, W, t, scratch), "overlap")
    _refused((src, dst, B, H, W, t, dst), "overlap")
    torch.cuda.synchronize()
    assert bool((dst == SENTINEL).all()) and bool((scratch == SENTINEL).all())
    # the Python entry refuses before any launch too
    before = _cabi.launch_count
    for bad_call in (lambda: jpeg.roundtrip_u8(src.float()), lambda: jpeg.roundtrip_u8(src[0]),
                     lambda: jpeg.roundtrip_u8(src[..., :2].contiguous()), lambda: jpeg.roundtrip_u8(src.cpu()),
                     lambda: jpeg.roundtrip_u8(src, 0), lambda: jpeg.roundtrip_u8(src, 101),
                     lambda: jpeg.roundtrip_u8(src, True)):
        with pytest.raises((TypeError, ValueError)):
            bad_call()
    assert _cabi.launch_count == before
    assert jpeg.roundtrip_u8(src[:0]).shape == (0, H, W, 3) and _cabi.launch_count == before


# ---- eval_step_fid(saved_as="jpeg") against the script's files
@pytest.fixture(scope="module")
def model():
    import omnitokenizer_b200 as ob
    from oracle import omni_oracle as oo
    from oracle import weights as W
    args = ob.canonical_args()
    m = ob.OmniTokenizer_VQGAN(args)
    m.load_state_dict(W.make_state_dict(oo.Config.from_args(args), 0), strict=False)
    m.codebook._need_init = False
    return m.to(DEV).eval()


@pytest.fixture(scope="module")
def inception():
    from oracle import fid_oracle as fo
    g = load_golden("fid_inception")
    sd = fo.make_state_dict(g["w_seed"])
    sd.update(g["bn"])
    return fid.FIDInception(sd, DEV)


def _saved_and_reopened(a: np.ndarray, side) -> np.ndarray:
    """vqgan_eval.py:204-220 for one image array and a .JPEG path: resize (if any), save, and pytorch-fid's reopen."""
    from PIL import Image
    img = Image.fromarray(a)
    if side is not None:
        img = img.resize((side, side), getattr(Image, "ANTIALIAS", Image.LANCZOS))
    f = io.BytesIO()
    img.save(f, format=Image.registered_extensions()[".jpeg"])
    f.seek(0)
    return np.asarray(Image.open(f).convert("RGB"))


@pytest.mark.parametrize("d", [None, 2, 3])
def test_eval_step_fid_jpeg_equals_saved_files(model, inception, d):
    from oracle import fid_oracle as fo
    images = [fo.image_bytes(s, 70 + i) for i, s in enumerate([(150, 200), (128, 128), (97, 131)])]
    resize = L.image_resize(128)
    usage = torch.zeros(8192, device=DEV)
    real_f, fake_f, vq_output = C.eval_step_fid(model, images, resize, inception, usage, infer_downsample=d,
                                                saved_as="jpeg")
    host = torch.stack([L.resize_u8(im, resize) for im in images])
    x = L.u8_normalize(host.unsqueeze(1), C.IMAGE_NORM)[:, :, 0]
    real_saved = ((x.permute(0, 2, 3, 1) + 0.5).numpy() * 255).astype(np.uint8)          # vqgan_eval.py:204-205
    fake_bytes, vq2 = C.eval_step_u8(model, host.to(DEV), None, C.IMAGE_NORM)
    fake_saved = fake_bytes[:, 0].cpu().numpy()                                          # :214-215
    side = None if d is None else 128 // d
    real_files = np.stack([_saved_and_reopened(a, side) for a in real_saved])
    fake_files = np.stack([_saved_and_reopened(a, side) for a in fake_saved])
    if d is None:
        assert not np.array_equal(fake_files, fake_saved)                               # JPEG changed the bytes
    assert torch.equal(real_f, inception.features(torch.from_numpy(real_files).to(DEV)).clone())
    assert torch.equal(fake_f, inception.features(torch.from_numpy(fake_files).to(DEV)).clone())
    assert torch.equal(vq_output["batch_usage"], vq2["batch_usage"]) and bool(usage.sum() > 0)
    # the default is the lossless format, which the round trip leaves out
    real_png, fake_png, _ = C.eval_step_fid(model, images, resize, inception, infer_downsample=d)
    assert not torch.equal(real_png, real_f) and not torch.equal(fake_png, fake_f)


def test_saved_format_of_the_shipped_datasets():
    assert C.saved_format("val/n01440764/ILSVRC2012_val_00000293.JPEG") == "jpeg"
    assert C.saved_format("CelebAMask-HQ/CelebA-HQ-img/10012.jpg") == "jpeg"
    assert C.saved_format("ffhq/00000.png") == "png"
