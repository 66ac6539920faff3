"""The FID oracle (oracle/fid_oracle.py) against the fixture the unmodified pytorch-fid InceptionV3 wrote, and
deliberately broken wirings of it landing far from the fixture."""
import os

import pytest
import torch

from oracle import fid_oracle as fo

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "fid_inception.pt")


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN)


@pytest.fixture(scope="module")
def sd(golden):
    sd = fo.make_state_dict(golden["w_seed"])
    assert fo.conv_fingerprint(sd) == golden["fingerprint"]
    sd.update(golden["bn"])
    return sd


def _u8(e):
    return fo.image_bytes(e["shape"], e["seed"])[None]


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


def test_fixture_shape(golden):
    assert len(golden["bn"]) == 2 * 94
    assert set(golden["images"]) == {"up_256", "up_128", "same_299", "down_320x480", "odd_97x131", "const_64x80"}
    for e in golden["images"].values():
        assert e["features"].shape == (2048,)


def test_oracle_matches_reference(golden, sd):
    for name, e in golden["images"].items():
        with torch.no_grad():
            got = fo.forward(sd, fo.preprocess(_u8(e)))[0]
        rel = _rel(got, e["features"])
        print(f"{name}: oracle vs reference {rel:.2e}")
        assert rel <= 1e-6, name


def test_preprocess_matches_reference(golden):
    for name, e in golden["images"].items():
        x = fo.preprocess(_u8(e))
        assert torch.equal(x.flatten()[e["pre_idx"]], e["pre_val"]), name


def test_endpoints_match(golden, sd):
    e = golden["images"]["up_256"]
    eps = {}
    with torch.no_grad():
        fo.forward(sd, fo.preprocess(_u8(e)), eps)
    for k, s in e["endpoints"].items():
        v = eps[k]
        assert float((v.flatten()[s["idx"]] - s["val"]).abs().max()) <= 1e-5 * float(s["val"].abs().max() + 1), k
        assert float((v.mean(dim=(0, 2, 3)) - s["channel_mean"]).abs().max()) <= 1e-5, k


@pytest.mark.parametrize("wiring", [dict(count_include_pad=True), dict(e2_avg=True), dict(eps=1e-5)])
def test_broken_network_wirings_are_far(golden, sd, wiring):
    e = golden["images"]["up_256"]
    with torch.no_grad():
        got = fo.forward(sd, fo.preprocess(_u8(e)), **wiring)[0]
    rel = _rel(got, e["features"])
    print(f"{wiring}: {rel:.2e}")
    assert rel > 1e-3


def test_align_corners_is_far(golden, sd):
    e = golden["images"]["down_320x480"]
    with torch.no_grad():
        got = fo.forward(sd, fo.preprocess(_u8(e), align_corners=True))[0]
    rel = _rel(got, e["features"])
    print(f"align_corners=True: {rel:.2e}")
    assert rel > 1e-3


def test_normalising_before_the_resize_changes_the_bits(golden):
    """2 x - 1 before the resize is the same function up to rounding (the bilinear weights sum to 1), so it shows in
    the preprocess bits rather than in the features."""
    for name in ("up_256", "down_320x480", "odd_97x131"):
        e = golden["images"][name]
        x = fo.preprocess(_u8(e), norm_first=True)
        assert not torch.equal(x.flatten()[e["pre_idx"]], e["pre_val"]), name
