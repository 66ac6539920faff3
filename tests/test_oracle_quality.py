"""The quality oracle (oracle/quality_oracle.py) against the fixture the unmodified calculate_psnr.py / calculate_ssim.py
and lpips.py wrote, and deliberately broken wirings of it landing far from the fixture."""
import os

import pytest
import torch

from oracle import quality_oracle as qo

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "quality.pt")


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN)


@pytest.fixture(scope="module")
def sd(golden):
    sd = qo.make_state_dict(golden["w_seed"])
    assert qo.fingerprint(sd) == golden["fingerprint"]
    return sd


def _pair(e):
    a, b = qo.frame_pair(e["spec"])
    return qo.to01(a)[None], qo.to01(b)[None]


def test_fixture_shape(golden):
    assert golden["taps"].dtype == torch.float64 and golden["taps"].shape == (11,)
    assert os.path.getsize(GOLDEN) < 1_000_000
    c = golden["cases"]
    assert c["same_64"]["psnr"] == 100 and c["same_64"]["ssim"] == 1.0 and c["same_64"]["lpips"] == 0.0
    assert c["one_byte_256"]["psnr"] == 100            # mse 7.8e-11 < 1e-10
    assert c["two_bytes_256"]["psnr"] < 100            # mse 1.6e-10


@pytest.mark.parametrize("name", ["noise_256", "noise_64", "noise_67x93", "min_ssim_11", "min_lpips_16", "same_64",
                                  "const_32", "one_byte_256", "two_bytes_256"])
def test_psnr_ssim_match_reference(golden, name):
    e = golden["cases"][name]
    a, b = _pair(e)
    an, bn = a[0].double().numpy(), b[0].double().numpy()
    assert abs(qo.psnr(an, bn) - e["psnr"]) <= 1e-12 * max(1.0, abs(e["psnr"]))
    assert abs(qo.ssim(an, bn, golden["taps"].numpy()) - e["ssim"]) <= 1e-11


def test_gaussian_close_to_cv2(golden):
    assert float((torch.from_numpy(qo.gaussian()) - golden["taps"]).abs().max()) <= 1e-16


@pytest.mark.parametrize("name", ["noise_64", "noise_67x93", "min_lpips_16", "same_64", "const_32"])
def test_lpips_matches_reference(golden, sd, name):
    e = golden["cases"][name]
    a, b = _pair(e)
    with torch.no_grad():
        per_tap = []
        v = float(qo.lpips(sd, a, b, per_tap=per_tap)[0])
    assert abs(v - e["lpips"]) <= 1e-6 * max(abs(e["lpips"]), 1e-3)
    assert torch.allclose(torch.stack([t[0] for t in per_tap]), e["lpips_taps"], rtol=1e-5, atol=1e-9)


def _ssim_err(golden, **kw):
    e = golden["cases"]["noise_64"]
    a, b = _pair(e)
    return abs(qo.ssim(a[0].double().numpy(), b[0].double().numpy(), **kw) - e["ssim"])


def test_wrong_ssim_wirings_are_caught(golden):
    assert _ssim_err(golden, taps=golden["taps"].numpy()) <= 1e-11
    assert _ssim_err(golden, taps=golden["taps"].numpy(), same=True) > 1e-4     # the "same" map, not the valid crop
    assert _ssim_err(golden, sigma=1.0) > 1e-4                                 # a wrong sigma


@pytest.mark.parametrize("wrong", [dict(scale_01=True), dict(pre_relu=True), dict(eps=0.0), dict(drop_tap=2),
                                   dict(drop_tap=4)],
                         ids=["scaling_on_01", "taps_before_relu", "no_eps", "missing_tap2", "missing_tap4"])
def test_wrong_lpips_wirings_are_caught(golden, sd, wrong):
    name = "const_32" if "eps" in wrong else "noise_64"
    e = golden["cases"][name]
    a, b = _pair(e)
    if "eps" in wrong:
        # a pixel whose features are all zero normalises to zero only through the 1e-10: kill relu1_2 (and with it every
        # later tap's dependence on the input) and the right head gives exactly 0, the one without the 1e-10 0 / 0
        dead = dict(sd)
        dead["net.slice1.2.bias"] = torch.full_like(sd["net.slice1.2.bias"], -1e4)
        with torch.no_grad():
            assert float(qo.lpips(dead, a, b)[0]) == 0.0
            assert torch.isnan(qo.lpips(dead, a, b, **wrong)).all()
            assert abs(float(qo.lpips(sd, a, b)[0]) - e["lpips"]) <= 1e-6 * abs(e["lpips"])
        return
    with torch.no_grad():
        v = float(qo.lpips(sd, a, b, **wrong)[0])
    assert abs(v - e["lpips"]) > 1e-3 * abs(e["lpips"])
