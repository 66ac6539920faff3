"""Host logic of omnitokenizer_b200.quality without a GPU: the LPIPS checkpoint key mapping and its named errors, the
value tables against the torch chain, the PSNR 100 rule, the result dicts against the suite's aggregation and every
refusal before a launch."""
import os

import numpy as np
import pytest
import torch

from omnitokenizer_b200 import consumers, quality
from omnitokenizer_b200.fid import byte_lut
from omnitokenizer_b200.fvd import real_byte_table
from omnitokenizer_b200.layout import U8Norm
from oracle import quality_oracle as qo

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "quality.pt")


@pytest.fixture(scope="module")
def sd():
    return qo.make_state_dict(3)


def _packed(model):
    return [u.w_hi + u.w_lo for units in model.units for u in units]


def test_taps_are_cv2s():
    assert torch.equal(quality.gaussian_taps(), torch.load(GOLDEN)["taps"])
    assert float((quality.gaussian_taps_formula() - quality.gaussian_taps()).abs().max()) <= 1e-16


def test_expected_keys_match_oracle(sd):
    assert set(quality.expected_keys()) == set(sd)
    for k, shape in quality.expected_keys().items():
        assert tuple(sd[k].shape) == shape


def test_checkpoint_prefix_and_layouts(sd):
    bare = quality.LPIPS(sd, device="cpu")
    ckpt = {"encoder.x.weight": torch.zeros(2), "image_discriminator.y": torch.zeros(1)}
    ckpt.update({"perceptual_model." + k: v for k, v in sd.items()})
    from_ckpt = quality.LPIPS(ckpt, device="cpu")
    tv = {f"features.{idx}.{f}": sd[f"net.slice{s}.{idx}.{f}"]
          for s, convs in enumerate(qo.VGG_SLICES, 1) for idx, _, _ in convs for f in ("weight", "bias")}
    tv["classifier.0.weight"] = torch.zeros(4, 4)
    tv.update({k: v for k, v in sd.items() if k.startswith("lin")})
    from_tv = quality.LPIPS(tv, device="cpu")
    for m in (from_ckpt, from_tv):
        assert all(torch.equal(x, y) for x, y in zip(_packed(m), _packed(bare)))
        assert all(torch.equal(x, y) for x, y in zip(m.lin, bare.lin))
        assert torch.equal(m.shift_scale, bare.shift_scale)
    # the checkpoint's own buffers are used, not the constants
    sd2 = dict(sd)
    sd2["scaling_layer.shift"] = sd["scaling_layer.shift"] + 0.25
    assert not torch.equal(quality.LPIPS(sd2, device="cpu").shift_scale, bare.shift_scale)
    # packed conv weights: K = (dh, dw, c), c padded to 4 for the RGB input
    u = bare.units[0][0]
    assert u.K == 64 and u.w_hi.shape == (128, 64)
    w = sd["net.slice1.0.weight"]
    assert torch.equal((u.w_hi + u.w_lo)[:64, :36].view(64, 3, 3, 4)[..., :3], w.permute(0, 2, 3, 1))


def test_named_key_errors(sd):
    bad = dict(sd)
    del bad["lin3.model.1.weight"]
    with pytest.raises(KeyError, match="lin3.model.1.weight"):
        quality.LPIPS(bad, device="cpu")
    bad = dict(sd)
    bad["net.slice3.12.weight"] = torch.zeros(256, 256, 1, 1)
    with pytest.raises(ValueError, match=r"net\.slice3\.12\.weight"):
        quality.LPIPS(bad, device="cpu")
    bad = dict(sd)
    bad["net.slice9.0.weight"] = torch.zeros(1)
    with pytest.raises(KeyError, match="slice9"):
        quality.LPIPS(bad, device="cpu")


def test_other_nets_refused(sd):
    with pytest.raises(NotImplementedError, match="alex"):
        quality.LPIPS(sd, device="cpu", net="alex")
    with pytest.raises(NotImplementedError, match="spatial"):
        quality.LPIPS(sd, device="cpu", spatial=True)


NORMS = [None, U8Norm("video_norm", (0.5,) * 3, (1.0,) * 3, max_test=True), U8Norm("image_norm", (0.5,) * 3, (1.0,) * 3)]


@pytest.mark.parametrize("norm", NORMS, ids=["plain", "video_norm", "image_norm"])
def test_input_table_bit_equal_to_torch_chain(sd, norm):
    shift, scale = sd["scaling_layer.shift"], sd["scaling_layer.scale"]
    tab = quality.input_table(shift.view(3), scale.view(3), norm)
    byt = torch.arange(256, dtype=torch.uint8).view(1, 256).expand(3, 256)
    reals = [byt] if norm is None else [real_byte_table(norm)[t].view(1, 256).expand(3, 256) for t in
                                       range(real_byte_table(norm).shape[0])]
    assert tab.shape == (len(reals), 3, 256)
    for t, r in enumerate(reals):
        x01 = r.float().div(255).view(1, 3, 16, 16)                       # ToTensor's byte / 255 of the saved byte
        want = ((x01 * 2 - 1) - shift) / scale                            # calculate_lpips.trans, ScalingLayer
        assert torch.equal(tab[t], want.view(3, 256))
        assert torch.equal(byte_lut(norm)[t], r[0].float() / 255)


def test_psnr_rule():
    n = 3 * 256 * 256
    d = 1 / 255
    one, two = torch.tensor([d * d], dtype=torch.float64), torch.tensor([2 * d * d], dtype=torch.float64)
    assert float(quality.psnr_from_sse(one, n)) == 100.0                 # mse 7.8e-11
    p2 = float(quality.psnr_from_sse(two, n))
    assert p2 < 100 and abs(p2 - qo.psnr(np.zeros(n), np.r_[np.zeros(n - 2), d, d])) < 1e-9
    assert float(quality.psnr_from_sse(torch.tensor([0.0]), n)) == 100.0
    s = torch.tensor([12.5], dtype=torch.float64)
    assert float(quality.psnr_from_sse(s, n)) == pytest.approx(20 * np.log10(1 / np.sqrt(12.5 / n)), rel=1e-15)


def _reference_aggregation(results, video_shape):
    """calculate_psnr.py / calculate_ssim.py / calculate_lpips.py's tail, restated."""
    results = np.array(results)
    value, std = {}, {}
    for t in range(results.shape[1]):
        value[t] = np.mean(results[:, t])
        std[t] = np.std(results[:, t])
    return {"value": value, "value_std": std, "video_setting": video_shape,
            "video_setting_name": "time, channel, heigth, width"}


def test_result_dict_matches_reference_aggregation():
    g = np.random.default_rng(3)
    per = g.random((5, 7))
    per[2, 3] = 100
    shape = torch.zeros(7, 3, 16, 16).shape
    got, want = quality.result_dict(per, shape), _reference_aggregation(per.tolist(), shape)
    assert got.keys() == want.keys() and got["video_setting"] == want["video_setting"]
    for k in ("value", "value_std"):
        assert list(got[k]) == list(range(7))
        assert all(got[k][t] == want[k][t] for t in range(7))


def _u8(*shape):
    return torch.zeros(*shape, dtype=torch.uint8)


@pytest.mark.parametrize("case,exc,match", [
    ((_u8(1, 2, 16, 16, 3), torch.zeros(1, 2, 16, 16, 3)), TypeError, "uint8"),
    ((_u8(1, 16, 16, 3), _u8(1, 16, 16, 3)), ValueError, "rank 5"),
    ((_u8(1, 2, 16, 16, 3), _u8(1, 2, 16, 17, 3)), ValueError, "differ in shape"),
    ((_u8(1, 2, 16, 16, 1), _u8(1, 2, 16, 16, 1)), ValueError, "3 channels"),
    ((_u8(1, 2, 10, 16, 3), _u8(1, 2, 10, 16, 3)), ValueError, "SSIM"),
    ((_u8(1, 2, 16, 16, 3), _u8(1, 2, 16, 16, 3)), ValueError, "CUDA"),
], ids=["dtype", "rank", "shape", "channels", "ssim_size", "host_frames"])
def test_frame_metrics_refusals(case, exc, match):
    with pytest.raises(exc, match=match):
        quality.frame_metrics(*case)


def test_lpips_size_refusal(sd):
    m = quality.LPIPS(sd, device="cpu")
    with pytest.raises(ValueError, match="LPIPS"):
        quality.frame_metrics(_u8(1, 1, 15, 64, 3), _u8(1, 1, 15, 64, 3), m)
    with pytest.raises(ValueError, match="LPIPS"):
        quality.calculate_lpips_vgg(torch.zeros(1, 1, 3, 15, 64), torch.zeros(1, 1, 3, 15, 64), m)


def test_per_channel_norm_refused():
    norm = U8Norm("per_channel", (0.4, 0.5, 0.6), (1.0, 1.0, 1.0))
    with pytest.raises(ValueError, match="per channel"):
        quality.frame_metrics(_u8(1, 1, 16, 16, 3), _u8(1, 1, 16, 16, 3), real_norm=norm)


@pytest.mark.parametrize("fn", [quality.calculate_psnr, quality.calculate_ssim])
def test_dropin_refusals(fn):
    with pytest.raises(ValueError, match="differ in shape"):
        fn(torch.zeros(1, 2, 3, 16, 16), torch.zeros(1, 2, 3, 16, 17))
    with pytest.raises(ValueError, match="3 channels"):
        fn(torch.zeros(1, 2, 1, 16, 16), torch.zeros(1, 2, 1, 16, 16))
    with pytest.raises(ValueError, match="11"):
        fn(torch.zeros(1, 2, 3, 16, 10), torch.zeros(1, 2, 3, 16, 10))
    with pytest.raises(TypeError, match="floating point"):
        fn(torch.zeros(1, 2, 3, 16, 16, dtype=torch.uint8), torch.zeros(1, 2, 3, 16, 16, dtype=torch.uint8))
    with pytest.raises(ValueError, match=r"\(B, T, C, H, W\)"):
        fn(torch.zeros(2, 3, 16, 16), torch.zeros(2, 3, 16, 16))


def test_eval_step_quality_refuses_before_forward():
    class Boom:
        def forward_u8(self, *a, **k):
            raise AssertionError("forward ran before the refusal")

    with pytest.raises(ValueError, match="SSIM"):
        consumers.eval_step_quality(Boom(), _u8(1, 9, 10, 10, 3))
    with pytest.raises(ValueError, match="3 channels"):
        consumers.eval_step_quality(Boom(), _u8(1, 9, 16, 16, 1))
    with pytest.raises(TypeError, match="uint8"):
        consumers.eval_step_quality(Boom(), torch.zeros(1, 9, 16, 16, 3))
    with pytest.raises(ValueError, match="per channel"):
        consumers.eval_step_quality(Boom(), _u8(1, 9, 16, 16, 3), norm=U8Norm("p", (0.4, 0.5, 0.6), (1.0,) * 3))


def test_chunking_keeps_conv_rows_in_range():
    assert quality.chunk_pairs(136, 256, 256, True) == 32          # 2 * 32 * 256^2 = 2^22 rows
    assert quality.chunk_pairs(136, 256, 256, False) == 136
    assert quality.chunk_pairs(3, 2048, 2048, True) == 1
    for P, H, W in ((136, 256, 256), (1000, 67, 93), (5, 1024, 1024)):
        n = quality.chunk_pairs(P, H, W, True)
        assert 1 <= n <= P and 2 * n * H * W <= max(quality.LPIPS_ROWS, 2 * H * W) <= quality.MAX_CONV_ROWS
    with pytest.raises(ValueError, match="rows"):
        quality._check_sizes(40000, 40000, 3, "x", True)
