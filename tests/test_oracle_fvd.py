"""The CPU oracle of the FVD feature network (oracle/i3d_oracle.py) against the reference fixture
tests/golden/fvd_i3d.pt (oracle/make_golden_fvd.py), and broken wirings that must land far from it."""
import os

import pytest
import torch

from oracle import i3d_oracle as io

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "fvd_i3d.pt")


@pytest.fixture(scope="module", autouse=True)
def threads():
    """fvd.py's preprocess runs in the script's main process, where torch is multi-threaded; its single-threaded
    bilinear kernel rounds differently."""
    n = torch.get_num_threads()
    torch.set_num_threads(max(n, 2))
    yield
    torch.set_num_threads(n)


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN)


@pytest.fixture(scope="module")
def sd(golden):
    sd = io.make_state_dict(golden["w_seed"])
    sd.update(golden["bn"])
    assert io.conv_fingerprint(sd) == golden["fingerprint"]
    return sd


def clip(e):
    shape = tuple(e["shape"]) + (3,)
    if e["seed"] is None:
        return torch.full(shape, 200, dtype=torch.uint8)[None]
    return torch.randint(0, 256, shape, generator=torch.Generator().manual_seed(e["seed"]), dtype=torch.uint8)[None]


def rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


def test_fixture_is_small(golden):
    assert os.path.getsize(GOLDEN) < 1 << 20
    assert set(golden["clips"]) == {"down_17x256", "up_9x64", "ucf_17x240x320", "odd_33x97x131", "const_9x80x96"}


@pytest.mark.parametrize("name", ["down_17x256", "up_9x64", "ucf_17x240x320", "odd_33x97x131", "const_9x80x96"])
def test_oracle_matches_fixture(golden, sd, name):
    e = golden["clips"][name]
    x = io.preprocess(clip(e).numpy())
    assert torch.equal(x.flatten()[e["pre_idx"]], e["pre_val"])
    eps = {}
    with torch.no_grad():
        logits = io.forward(sd, x, eps)[0]
    assert rel(logits, e["logits"]) <= 2e-6
    for k, s in e.get("endpoints", {}).items():
        got = io.endpoint_summary(eps[k], 0)
        assert torch.allclose(got["channel_mean"], s["channel_mean"], rtol=1e-5, atol=1e-6), k
        assert torch.allclose(eps[k].flatten()[s["idx"]], s["val"], rtol=1e-5, atol=1e-6), k


def test_endpoints_are_order_one(golden):
    for k, s in golden["clips"]["down_17x256"]["endpoints"].items():
        m = float(s["channel_mean"].abs().max())
        assert 0.05 < m < 20, (k, m)


def test_frechet_distance_matches_fixture(golden):
    fd = golden["fd"]
    assert abs(float(io.frechet_distance(fd["x1"], fd["x2"])) / float(fd["value"]) - 1) < 1e-6


def test_normalising_before_the_resize_changes_the_bits(golden):
    """Bilinear weights sum to one, so the broken order only rounds differently: the stored preprocess sample sees it."""
    for e in golden["clips"].values():
        if e["seed"] is None:
            continue
        x = io.preprocess(clip(e).numpy(), norm_first=True)
        assert int((x.flatten()[e["pre_idx"]] != e["pre_val"]).sum()) > 50


@pytest.mark.parametrize("broken", ["symmetric_pad", "bn_eps_1e-3", "branch_order"])
def test_broken_wiring_lands_far(golden, sd, broken):
    far = 0.0
    for name in ("up_9x64", "odd_33x97x131", "const_9x80x96"):
        e = golden["clips"][name]
        x = io.preprocess(clip(e).numpy())
        kw = {"symmetric_pad": dict(symmetric=True), "bn_eps_1e-3": dict(eps=1e-3),
              "branch_order": dict(branch_order=(0, 2, 1, 3))}.get(broken, {})
        with torch.no_grad():
            y = io.forward(sd, x, **kw)[0]
        # symmetric padding also changes the feature map's size: the head then leaves extra dimensions
        far = max(far, rel(y, e["logits"]) if y.shape == e["logits"].shape else float("inf"))
    assert far > 1e-3, far
