"""CPU tests: the oracle on architecture flags other than the canonical ones, against the reference's outputs recorded by
oracle/make_golden_flags.py (tests/golden/flags.pt), and a sensitivity check per row: the oracle with the row's distinguishing
flag reverted (or its wiring broken the way an engine could break it) lands far from the fixture, so a fixture cannot agree
with an engine that ignores the flag."""
import dataclasses
import os

import pytest
import torch

from oracle import omni_oracle as oo
from tests.util import GOLDEN, check_sub, flags_namespace, flags_setup

ROWS = ["backfill", "stage1", "attn_causal_only", "peg_causal_only", "blocks", "ff2", "ff3", "nol2"]
PIX_TOL = 2e-6


def flags_golden():
    return torch.load(os.path.join(GOLDEN, "flags.pt"), weights_only=False)


def _share_window_bias(sd, cfg):
    """every window layer reads the bias table of the first window layer of its transformer"""
    sd = dict(sd)
    for pre, block in (("encoder.enc_spatial_transformer", cfg.enc_block), ("decoder.dec_spatial_transformer", cfg.dec_block)):
        w = [i for i, b in enumerate(block) if b == "w"]
        for i in w[1:]:
            sd[f"{pre}.layers.{i}.1.relative_position_bias_table"] = sd[f"{pre}.layers.{w[0]}.1.relative_position_bias_table"]
    return sd


def _swap_geglu_halves(sd, cfg):
    """gelu applied to the value half and the gate half passed through: a GEGLU packed the wrong way round"""
    sd = dict(sd)
    for k in [k for k in sd if k.endswith(".3.1.weight")]:
        w = sd[k]
        inner = w.shape[0] // 2
        sd[k] = torch.cat([w[inner:], w[:inner]])
    return sd


def _cfg(**over):
    return lambda sd, cfg: (sd, dataclasses.replace(cfg, **over))


def _sd(fn):
    return lambda sd, cfg: (fn(sd, cfg), cfg)


# row -> what the fixture must tell apart from it: the row's flags reverted to canonical, one at a time
SENSITIVITY = {
    "backfill": {"rope": _cfg(spatial_pos="rope"), "causal_peg": _cfg(causal_in_peg=True),
                 "causal_attn": _cfg(causal_in_temporal_transformer=True), "l2": _cfg(l2_code=True)},
    "stage1": {"rope": _cfg(spatial_pos="rope")},
    "attn_causal_only": {"causal_peg": _cfg(causal_in_peg=True),
                         "swapped": _cfg(causal_in_peg=True, causal_in_temporal_transformer=False)},
    "peg_causal_only": {"causal_attn": _cfg(causal_in_temporal_transformer=True),
                        "swapped": _cfg(causal_in_peg=False, causal_in_temporal_transformer=True)},
    "blocks": {"shared_window_bias": _sd(_share_window_bias)},
    "ff2": {"geglu_swapped": _sd(_swap_geglu_halves)},
    "ff3": {"geglu_swapped": _sd(_swap_geglu_halves)},
    "nol2": {"l2": _cfg(l2_code=True)},
}


def test_fixture_covers_every_row():
    g = flags_golden()
    assert sorted(k for k in g if k != "torch") == sorted(ROWS) == sorted(SENSITIVITY)


def test_rows_differ_from_canonical_as_described():
    """Each row's Namespace reads as the model its name says (the back-fills of an old checkpoint included)."""
    g = flags_golden()
    canon = dataclasses.asdict(oo.Config())
    want = {"backfill": dict(enc_block="tttt", twod_window_size=4, spatial_pos="rel",
                             causal_in_temporal_transformer=False, causal_in_peg=False, l2_code=False),
            "stage1": dict(temporal_patch_size=2, spatial_pos="rel"),
            "attn_causal_only": dict(causal_in_peg=False),
            "peg_causal_only": dict(causal_in_temporal_transformer=False),
            "blocks": dict(enc_block="wtwt", dec_block="twwt", temporal_depth=2),
            "ff2": dict(ff_mult=2.0), "ff3": dict(ff_mult=3.0),
            "nol2": dict(l2_code=False)}
    for name in ROWS:
        cfg, _, _ = flags_setup(g[name])
        diff = {k: v for k, v in dataclasses.asdict(cfg).items() if v != canon[k] and k != "resolution"}
        assert diff == want[name], (name, diff)
    assert oo.Config.from_args(flags_namespace(g["ff2"])).ff_inner == 682
    assert oo.Config.from_args(flags_namespace(g["ff3"])).ff_inner == 1024


@pytest.mark.parametrize("name", ROWS)
def test_oracle_matches_flags_golden(name):
    row = flags_golden()[name]
    cfg, sd, xs = flags_setup(row)
    for x, r in zip(xs, row["inputs"]):
        is_image = x.ndim == 4
        with torch.no_grad():
            emb, idx = oo.encode(sd, cfg, x, include_embeddings=True)
            rec = oo.decode(sd, cfg, idx, is_image)
        mism = int((idx != r["idx"].long()).sum())
        assert mism == 0, f"{name} {tuple(x.shape)}: {mism}/{idx.numel()} code indices differ from the reference"
        assert (emb - r["emb"]).abs().max().item() <= 1e-6
        err = check_sub(r["rec"], rec, PIX_TOL, f"{name} {tuple(x.shape)} reconstruction")
        print(f"{name} {tuple(x.shape)}: 0/{idx.numel()} index mismatches, max |dpixel| {err:.2e}")


@pytest.mark.parametrize("name", ROWS)
def test_flags_golden_is_sensitive_to_the_row_flags(name):
    row = flags_golden()[name]
    cfg, sd, xs = flags_setup(row)
    x, r = xs[0], row["inputs"][0]
    is_image = x.ndim == 4
    for label, revert in SENSITIVITY[name].items():
        sd2, cfg2 = revert(sd, cfg)
        with torch.no_grad():
            idx = oo.encode(sd2, cfg2, x)
            rec = oo.decode(sd2, cfg2, r["idx"].long(), is_image)
        mism = int((idx != r["idx"].long()).sum())
        err = check_sub(r["rec"], rec, float("inf"), label)
        print(f"{name} / {label}: {mism}/{idx.numel()} codes differ, max |dpixel| {err:.2e}")
        assert mism > 0 or err > 1e-2, f"{name}: the fixture does not tell the row from '{label}'"
