"""The Inception Score oracle against the reference fixture (tests/golden/is_inception.pt, written by
oracle/make_golden_is.py from the unmodified calculate_is.py with torchvision's Inception3): the probabilities bit for
bit, the scores to float64 rounding, and each broken wiring caught."""
import os

import numpy as np
import pytest
import torch

from oracle import fid_oracle as fo
from oracle import is_oracle as io

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "is_inception.pt")


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN, weights_only=False)


@pytest.fixture(scope="module")
def sd(golden):
    s = io.fixture_state_dict(golden)
    assert fo.conv_fingerprint(s) == golden["fingerprint"]
    return s


def test_fixture_cases_are_the_oracle_cases(golden):
    assert list(golden["cases"]) == list(io.CASES)
    for name, spec in io.CASES.items():
        assert golden["cases"][name]["spec"] == spec


@pytest.mark.parametrize("name", list(io.CASES))
def test_oracle_equals_reference(golden, sd, name):
    g = golden["cases"][name]
    spec = g["spec"]
    probs = io.case_probabilities(sd, spec)
    assert torch.equal(probs, g["probs"])
    mean, std = io.inception_score(g["probs"].double().numpy(), spec["splits"])
    assert abs(mean - g["mean"]) <= 1e-12 * g["mean"]
    assert abs(std - g["std"]) <= 1e-12 * g["mean"]


def test_preprocess_samples(golden):
    for name, g in golden["cases"].items():
        spec = g["spec"]
        x, _ = io.case_input(spec)
        pre = torch.cat([io.preprocess(b, spec.get("resize", True)) for b in io.case_batches(spec, x)])
        assert tuple(pre.shape) == g["pre_shape"]
        assert torch.equal(pre.flatten()[g["pre_idx"]], g["pre_val"]), name


def test_u8_case_is_bytes_over_255():
    x, u8 = io.case_input(io.CASES["calc_u8_48x64"])
    assert torch.equal(x, u8.permute(0, 1, 4, 2, 3).float() / 255)


def _first_clip(golden):
    g = golden["cases"]["calc_up64"]
    x, _ = io.case_input(g["spec"])
    return x[0], g["probs"][:x.shape[1]]


@pytest.mark.parametrize("wiring", [dict(count_include_pad=False), dict(e2_avg=False), dict(align_corners=True),
                                    dict(softmax_dim=0)],
                         ids=["avg_without_padding", "max_pool_in_Mixed_7c", "align_corners", "softmax_dim0"])
def test_broken_network_wiring_is_caught(golden, sd, wiring):
    x, ref = _first_clip(golden)
    with torch.no_grad():
        bad = io.probabilities(sd, x, True, **wiring)
    assert float((bad - ref).abs().max()) > 1e-4


@pytest.mark.parametrize("wiring,case", [(dict(renormalise=False), "calc_up64"),
                                         (dict(keep_leftover=True), "calc_n7_splits3")],
                         ids=["entropy_without_renormalising", "leftover_rows_kept"])
def test_broken_score_wiring_is_caught(golden, wiring, case):
    g = golden["cases"][case]
    mean, _ = io.inception_score(g["probs"].double().numpy(), g["spec"]["splits"], **wiring)
    assert abs(mean - g["mean"]) > 1e-9 * g["mean"]
