"""vqgan_eval.py's --infer_downsample and --replacewithgt without a GPU: the host twins of omt_eval_downsample and of the
LANCZOS resize reproduce tests/golden/eval_downsample.pt byte for byte, the LANCZOS tables equal live Pillow, and every
refusal of the eval steps happens before any launch."""
import numpy as np
import pytest
import torch

from omnitokenizer_b200 import _cabi, consumers, downsample
from omnitokenizer_b200 import layout as L
from tests.util import load_golden


@pytest.fixture(scope="module")
def fx():
    return load_golden("eval_downsample")


def _real_twin(u8, d, one_thread, norm=consumers.VIDEO_NORM):
    sel = (u8.reshape(u8.shape[0], -1).amax(dim=1) <= 1).long().numpy() if norm.max_test else None
    return L.downsample_clips(u8, d, one_thread, downsample.real_value_table(norm), sel)


def test_fixture_covers_both_kernel_forms(fx):
    forms = set()
    for case in fx["video"]:
        B, T, H, W = fx["clips"][case["clip"]]["shape"]
        g = L.downsample_geometry(H, W, case["d"])
        forms.add(L.clip_interp_form(g, case["one_thread"]))
        assert tuple(case["real"].shape) == (B, T, g.rh, g.rw, 3)
    assert forms == {L.INTERP_SEPARABLE, L.INTERP_WEIGHTS}
    assert {v["d"] for v in fx["video"]} == {2, 3, 4}


def test_host_twin_equals_the_script(fx):
    for case in fx["video"] + fx["replace"]:
        c = fx["clips"][case["clip"]]
        d, one = case["d"], case["one_thread"]
        real = _real_twin(c["u8"], d, one)
        fake = L.downsample_clips(c["recons"], d, one)
        k = case.get("k", 0)
        fake[:, :k] = real[:, :k]
        assert torch.equal(real, case["real"]), (c["shape"], d, one)
        assert torch.equal(fake, case["fake"]), (c["shape"], d, one, k)


def test_replacewithgt_cases_swap_exactly_k_frames(fx):
    base = {(v["clip"], v["d"], v["one_thread"]): v for v in fx["video"]}
    for case in fx["replace"]:
        plain = base[(case["clip"], case["d"], case["one_thread"])]
        k = case["k"]
        assert torch.equal(case["fake"][:, :k], plain["real"][:, :k])
        assert torch.equal(case["fake"][:, k:], plain["fake"][:, k:])
        assert not torch.equal(plain["fake"][:, :max(k, 1)], plain["real"][:, :max(k, 1)])


def test_host_lanczos_equals_the_script(fx):
    im = fx["images"]
    real_bytes = downsample.real_value_table(consumers.IMAGE_NORM)
    real = L.downsample_clips(im["u8"].unsqueeze(1), 1, True, real_bytes)[:, 0]          # the saved input's bytes
    fake = L.downsample_clips(im["recons"].unsqueeze(2), 1, True)[:, 0]
    for d, (want_real, want_fake) in im["out"].items():
        rz = L.eval_downsample_resize(im["res"], d)
        assert torch.equal(torch.stack([L.resize_u8(x, rz) for x in real]), want_real), d
        assert torch.equal(torch.stack([L.resize_u8(x, rz) for x in fake]), want_fake), d


@pytest.mark.parametrize("src, dst", [((64, 64), (21, 21)), ((37, 53), (9, 13)), ((5, 7), (11, 3)), ((1, 1), (3, 3)),
                                      ((301, 11), (7, 5)), ((128, 128), (32, 32)), ((255, 99), (51, 33))])
def test_lanczos_tables_equal_pillow(src, dst):
    Image = pytest.importorskip("PIL.Image")
    g = torch.Generator().manual_seed(src[0] * 1000 + dst[1])
    img = torch.randint(0, 256, src + (3,), generator=g, dtype=torch.uint8)
    want = np.asarray(Image.fromarray(img.numpy()).resize((dst[1], dst[0]), Image.LANCZOS))
    assert torch.equal(L.resize_u8(img, L.U8Resize(dst, "antialias")), torch.from_numpy(want.copy()))


def test_lanczos_reaches_past_the_old_tap_counts():
    bounds, coeffs = L.resample_coeffs(256, 64, "antialias")       # d = 4: support 3 * 4 -> 25 taps
    assert coeffs.shape[1] == 25 and int(bounds[:, 1].max()) == 24
    assert all(abs(int(k.sum()) - (1 << 22)) <= 25 for k in coeffs)


def test_real_value_table_is_the_normalised_value_plus_half():
    t = downsample.real_value_table(consumers.VIDEO_NORM)
    assert t.shape == (2, 256) and t.dtype == torch.float32
    assert torch.equal(t[0], (torch.arange(256).float() / 255.0 - 0.5) + 0.5)
    assert torch.equal(t[1], torch.arange(256).float() - 0.5 + 0.5)
    with pytest.raises(ValueError, match="per channel"):
        downsample.real_value_table(L.U8Norm("x", (0.1, 0.2, 0.3), (1.0, 1.0, 1.0)))


class _NoLaunch:
    """A model / network whose every use fails the test: a refusal must come first."""

    device = torch.device("cuda", 0)

    def __getattr__(self, name):
        raise AssertionError(f"touched {name} before refusing")


class _I3D(_NoLaunch):
    check_frames = staticmethod(lambda frames: None)


@pytest.mark.parametrize("kw, err, match", [
    (dict(infer_downsample=0), ValueError, "infer_downsample"),
    (dict(infer_downsample=-2), ValueError, "infer_downsample"),
    (dict(infer_downsample=1.5), TypeError, "infer_downsample"),
    (dict(infer_downsample=2.0), TypeError, "infer_downsample"),
    (dict(infer_downsample=64), ValueError, "infer_downsample"),
    (dict(replacewithgt=-1), ValueError, "replacewithgt"),
    (dict(replacewithgt=10), ValueError, "replacewithgt"),
    (dict(replacewithgt=1.0), TypeError, "replacewithgt"),
    (dict(replacewithgt=2, sequence_length=16), ValueError, "sequence_length"),
])
def test_fvd_refusals_before_any_launch(kw, err, match):
    frames = torch.zeros(2, 9, 32, 32, 3, dtype=torch.uint8)
    n0 = _cabi.launch_count
    with pytest.raises(err, match=match):
        consumers.eval_step_fvd(_NoLaunch(), frames, _I3D(), **kw)
    assert _cabi.launch_count == n0


@pytest.mark.parametrize("d, err", [(0, ValueError), (3.0, TypeError), (65, ValueError), (True, TypeError)])
def test_fid_refusals_before_any_launch(d, err):
    images = [torch.zeros(64, 64, 3, dtype=torch.uint8)]
    n0 = _cabi.launch_count
    with pytest.raises(err, match="infer_downsample"):
        consumers.eval_step_fid(_NoLaunch(), images, L.image_resize(64), _NoLaunch(), infer_downsample=d)
    assert _cabi.launch_count == n0


def test_lanczos_preset():
    assert L.eval_downsample_resize(256, 2) == L.U8Resize((128, 128), "antialias")
    assert L.eval_downsample_resize(256, 3).size == (85, 85)
    L.check_resize(L.eval_downsample_resize(64, 4))
