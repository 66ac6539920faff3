"""The video-metric suite's FVD without a GPU: the oracle preprocesses against the reference's hashes, the oracle's
StyleGAN-V forward against the live torchscript, the key map, the pad / ceil_mode equivalence, fvd_external's frame
selection, the result dict and the refusals."""
import hashlib
import os

import pytest
import torch

from omnitokenizer_b200 import _cabi, consumers, fvd, quality
from oracle import fvd_suite_oracle as so
from oracle import i3d_oracle as io

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "fvd_suite.pt")
TORCHSCRIPT = os.path.join(os.environ.get("OMT_REFERENCE_ROOT", "/root/reference"), "evaluation",
                           "common_metrics_on_video_quality", "fvd", "styleganv", "i3d_torchscript.pt")
needs_ref = pytest.mark.skipif(not os.path.isfile(TORCHSCRIPT), reason="reference tree not present")


def sha(t):
    return hashlib.sha256(t.contiguous().numpy().tobytes()).hexdigest()


@pytest.mark.parametrize("method", ["styleganv", "videogpt"])
def test_oracle_preprocess_matches_reference_hashes(method):
    fn = so.preprocess_styleganv if method == "styleganv" else so.preprocess_videogpt
    for name, case in torch.load(GOLDEN)["preprocess"].items():
        v = torch.rand(case["shape"], generator=torch.Generator().manual_seed(case["seed"]))
        assert sha(fn(v, case["shape"][1])) == case[method], name


@needs_ref
def test_oracle_forward_matches_torchscript():
    net = torch.jit.load(TORCHSCRIPT).eval()
    x = torch.rand(1, 3, 10, 224, 224, generator=torch.Generator().manual_seed(3)) * 2 - 1
    with torch.no_grad():
        ref = net(x, rescale=False, resize=False, return_features=True)
        got = so.forward_styleganv(net.state_dict(), x)
    assert float((got - ref).abs().max()) <= 1e-4 * float(ref.abs().max())


@needs_ref
def test_key_map_covers_the_torchscript():
    module = torch.jit.load(TORCHSCRIPT)
    sd = module.state_dict()
    assert len(sd) == 344
    mapped = fvd.styleganv_state_dict(sd)
    assert len(mapped) == 344
    assert {k for k in mapped if not k.endswith("num_batches_tracked")} == set(fvd.expected_keys())
    assert so.pytorch_i3d_keys(sd).keys() == {k for k in mapped if not k.endswith("num_batches_tracked")}
    assert fvd._scripted_pads(module) == {k: v[2] for k, v in fvd.STYLEGANV_PADS.items()}


def test_key_map_refuses_unknown_keys():
    with pytest.raises(KeyError):
        fvd.styleganv_key("mixed_3b.branch_4.conv3d.weight")
    with pytest.raises(KeyError):
        fvd.styleganv_key("conv3d_9z.conv3d.weight")


@pytest.mark.parametrize("T", range(9, 65))
def test_pad_tables_are_same_padding(T):
    fvd.check_styleganv_pads(T)


def test_pad_check_catches_a_wrong_table():
    pads = {k: v[2] for k, v in fvd.STYLEGANV_PADS.items()}
    pads["MaxPool3d_4a_3x3"] = ((0, 1, 0, 1, 1, 1), (0, 1, 0, 1, 1, 1))
    with pytest.raises(ValueError, match="MaxPool3d_4a_3x3"):
        fvd.check_styleganv_pads(16, pads=pads)
    with pytest.raises(ValueError, match="head"):
        fvd.check_styleganv_pads(8)


@pytest.mark.parametrize("n,frames,sampling,want", [
    (17, 17, "center", range(17)), (30, 17, "center", range(7, 24)), (30, 16, "center", range(7, 23)),
    (31, 16, "center", range(7, 23)), (31, 17, "center", range(7, 24)), (30, 17, "first", range(17)),
    (30, 17, "last", range(13, 30))])
def test_fvd_external_indices(n, frames, sampling, want):
    assert list(consumers.fvd_external_indices(n, frames, sampling)) == list(want)


def test_fvd_external_refusals():
    with pytest.raises(ValueError, match="fewer"):
        consumers.fvd_external_indices(16, 17)
    with pytest.raises(ValueError, match="sampling"):
        consumers.fvd_external_indices(20, 17, "middle")


def test_suite_geometry():
    for h, w in ((64, 64), (240, 320), (320, 240), (97, 131)):
        rh, rw = so.target_size(h, w)
        assert fvd.suite_geometry(h, w) == (rh, rw, (rh - 224) // 2, (rw - 224) // 2)


class _Net(fvd.I3D):
    """An I3D object without weights: enough for the checks calculate_fvd makes before any launch."""

    def __init__(self, variant):
        self.variant, self.device = variant, torch.device("cuda", 0)


def test_short_clips_give_an_empty_value():
    n0 = _cabi.launch_count
    r = quality.calculate_fvd(torch.rand(2, 9, 1, 32, 48), torch.rand(3, 9, 3, 40, 40), "cuda", "styleganv",
                              i3d=_Net("styleganv"))
    assert r == {"value": {}, "video_setting": torch.Size([2, 3, 9, 32, 48]),
                 "video_setting_name": "batch_size, channel, time, heigth, width"}
    r = quality.calculate_fvd(torch.zeros(2, 5, 32, 48, 3, dtype=torch.uint8), torch.rand(1, 9, 3, 8, 8), "cuda",
                              "videogpt", i3d=_Net("videogpt"))
    assert r["value"] == {} and r["video_setting"] == torch.Size([2, 3, 5, 32, 48])
    assert _cabi.launch_count == n0


@pytest.mark.parametrize("args,kw,err", [
    ((torch.rand(2, 12, 3, 8, 8).double(), torch.rand(2, 12, 3, 8, 8)), {}, TypeError),
    ((torch.rand(2, 12, 3, 8), torch.rand(2, 12, 3, 8, 8)), {}, ValueError),
    ((torch.rand(2, 12, 2, 8, 8), torch.rand(2, 12, 3, 8, 8)), {}, ValueError),
    ((torch.zeros(2, 12, 8, 8, 4, dtype=torch.uint8), torch.rand(2, 12, 3, 8, 8)), {}, ValueError),
    ((torch.rand(2, 12, 3, 8, 8), torch.rand(2, 11, 3, 8, 8)), {}, ValueError),
    ((torch.rand(2, 12, 3, 8, 8), torch.rand(2, 12, 3, 8, 8)), {"method": "tf"}, ValueError),
    ((torch.rand(2, 12, 3, 8, 8), torch.rand(2, 12, 3, 8, 8)), {"method": "videogpt"}, ValueError),
    ((torch.rand(2, 12, 3, 8, 8), torch.rand(2, 12, 3, 8, 8)), {"i3d": None}, TypeError),
])
def test_refusals(args, kw, err):
    kw = {"i3d": _Net("styleganv"), **kw}
    n0 = _cabi.launch_count
    with pytest.raises(err):
        quality.calculate_fvd(*args, "cuda", **kw)
    assert _cabi.launch_count == n0


def test_distances_follow_their_methods():
    g = torch.Generator().manual_seed(0)
    a, b = torch.randn(6, 20, generator=g, dtype=torch.float64), torch.randn(5, 20, generator=g, dtype=torch.float64)
    assert quality.frechet_distance_videogpt(a, b) == pytest.approx(float(fvd.frechet_distance(a, b)), rel=1e-12)
    one = quality.frechet_distance_videogpt(a[:1], b[:1])
    assert one == pytest.approx(float(((a[0] - b[0]) ** 2).sum()), rel=1e-12)
    assert quality.frechet_distance_styleganv(a[:1].numpy(), b[:1].numpy()) == pytest.approx(one, rel=1e-12)
    ref = float(io.frechet_distance(a, b))
    assert quality.frechet_distance_styleganv(a.numpy(), b.numpy()) == pytest.approx(ref, rel=1e-6)
