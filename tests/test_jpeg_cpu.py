"""The JPEG round trip of vqgan_eval.py's img.save(path) for .jpg / .JPEG datasets, on the host: oracle/jpeg_oracle.py
against Pillow run live, byte for byte, on the seeded grid; jpeg.quant_tables against the tables Pillow writes;
tests/golden/jpeg_roundtrip.pt against Pillow; five broken variants of the chain that must lose Pillow's bytes; and
consumers.saved_format's extension rule."""
import numpy as np
import pytest
import torch

from oracle import jpeg_oracle as J
from oracle.make_golden_jpeg import pillow_roundtrip, sha, versions
from omnitokenizer_b200 import consumers as C
from omnitokenizer_b200 import jpeg
from tests.util import load_golden

GRID = J.grid()
_upsample_chroma = J.upsample_chroma


def _mismatches(cases=GRID):
    bad = []
    for H, W, q, kind, seed in cases:
        x = J.content(kind, H, W, seed)
        if not np.array_equal(J.roundtrip(x, q), pillow_roundtrip(x, q)[0]):
            bad.append((H, W, q, kind, seed))
    return bad


def test_grid_covers_the_edges():
    shapes = {(H, W) for H, W, *_ in GRID}
    assert {(h, w) for h in range(1, 6) for w in range(1, 6)} <= shapes
    assert {(85, 85), (255, 257), (256, 256)} <= shapes
    assert any(H % 2 and not W % 2 for H, W in shapes) and any(W % 2 and not H % 2 for H, W in shapes)
    assert {q for *_, q, _, _ in GRID} >= {1, 100} and len({q for *_, q, _, _ in GRID}) > 60
    assert {k for *_, k, _ in GRID} == set(J.KINDS)
    assert max(max(H, W) for H, W in shapes if (H, W) not in {(255, 257), (256, 256)}) <= 99


def test_oracle_equals_pillow():
    bad = _mismatches()
    assert not bad, f"{len(bad)} of {len(GRID)} cases differ from Pillow, first {bad[:5]}"


@pytest.mark.parametrize("q", range(1, 101))
def test_quant_tables_equal_pillow(q):
    _, tables = pillow_roundtrip(np.zeros((8, 8, 3), np.uint8), q)
    assert np.array_equal(jpeg.quant_tables(q), tables)
    assert np.array_equal(J.quant_tables(q), tables)
    assert jpeg.quant_tables(q).dtype == np.uint16


@pytest.mark.parametrize("q", [0, 101, -5, 75.0, True, "75", None])
def test_quality_refused(q):
    with pytest.raises(ValueError, match="quality"):
        jpeg.quant_tables(q)


def test_golden_agrees_with_live_pillow():
    g = load_golden("jpeg_roundtrip")
    made_with = f"golden made with {g['versions']}, Pillow here is {versions()}"
    assert torch.equal(g["tables"], torch.from_numpy(np.stack([jpeg.quant_tables(q) for q in range(1, 101)])).int())
    assert [(c["H"], c["W"], c["quality"], c["kind"], c["seed"]) for c in g["cases"]] == GRID
    small = 0
    for c in g["cases"]:
        x = J.content(c["kind"], c["H"], c["W"], c["seed"])
        assert sha(x) == c["input_sha"], "the seeded input differs from the golden's"
        y, _ = pillow_roundtrip(x, c["quality"])
        assert sha(y) == c["output_sha"], (c["H"], c["W"], c["quality"], c["kind"], made_with)
        if "output" in c:
            small += 1
            assert np.array_equal(c["output"].numpy(), y)
    assert small >= 40


# ---- broken variants: each must lose Pillow's bytes somewhere on the grid
def _downsample_padded_rows(padded, H):
    """rule (a) replaced: the padded image rows are downsampled like real ones."""
    s = padded[0::2, 0::2] + padded[0::2, 1::2] + padded[1::2, 0::2] + padded[1::2, 1::2]
    return (s + np.where(np.arange(s.shape[1]) % 2 == 0, 1, 2)) >> 2


def _always_fancy(plane, H, W):
    """rule (b) dropped: fancy upsampling at every width."""
    ch, cw = -(-H // 2), -(-W // 2)
    c = plane[:ch, :cw]
    return J.fancy_upsample(c, np.concatenate([c[:1], c[:-1]]), np.concatenate([c[1:], c[-1:]]))[:H, :W]


def _context_from_padding(plane, H, W):
    """the bottom row's context taken from the decoded padding row below it (where there is one) instead of the edge
    row."""
    ch, cw = -(-H // 2), -(-W // 2)
    if cw <= 2 or ch == plane.shape[0]:
        return _upsample_chroma(plane, H, W)
    c = plane[:ch, :cw]
    return J.fancy_upsample(c, np.concatenate([c[:1], c[:-1]]), plane[1:ch + 1, :cw])[:H, :W]


def _truncating_quantize(coef, qt):
    d = (8 * qt).reshape(8, 8)
    return np.sign(coef) * (np.abs(coef) // d)


MUTANTS = {
    "rule_a_padded_rows": [("downsample_chroma", _downsample_padded_rows)],
    "rule_b_dropped": [("upsample_chroma", _always_fancy)],
    "biases_swapped": [("EVEN_BIAS", 7), ("ODD_BIAS", 8)],
    "truncating_quantisation": [("quantize", _truncating_quantize)],
    "context_from_padding": [("upsample_chroma", _context_from_padding)],
}


@pytest.mark.parametrize("name", sorted(MUTANTS))
def test_mutant_loses_pillows_bytes(name, monkeypatch):
    for attr, value in MUTANTS[name]:
        monkeypatch.setattr(J, attr, value)
    assert _mismatches(), f"the {name} variant still matches Pillow on the whole grid"


# ---- the script's format rule
@pytest.mark.parametrize("path, fmt", [
    ("val/n01440764/ILSVRC2012_val_00000293.JPEG", "jpeg"),        # eval_image_inet.sh
    ("CelebAMask-HQ/CelebA-HQ-img/10012.jpg", "jpeg"),             # eval_image_face.sh, CelebA-HQ
    ("ffhq/images1024x1024/00000.png", "png"),                     # eval_image_face.sh, FFHQ
    ("a/b.PNG", "png"), ("x.jpe", "jpeg"), ("x.JFIF", "jpeg"), ("dir.v2/x.Jpeg", "jpeg"),
])
def test_saved_format(path, fmt):
    assert C.saved_format(path) == fmt
    import pathlib
    assert C.saved_format(pathlib.PurePosixPath(path)) == fmt


@pytest.mark.parametrize("path", ["x.webp", "x.tif", "x.bmp", "noext", "x.jpg.gz"])
def test_saved_format_refuses_other_extensions(path):
    import os
    ext = os.path.splitext(path)[1].lower()
    with pytest.raises(NotImplementedError, match=repr(ext)):
        C.saved_format(path)


class _NoLaunch:
    def __getattr__(self, name):
        raise AssertionError(f"{name} used before the argument checks")


@pytest.mark.parametrize("saved_as", ["jpg", "JPEG", None, "webp"])
def test_eval_step_fid_refuses_unknown_format(saved_as):
    with pytest.raises(ValueError, match="saved_as"):
        C.eval_step_fid(_NoLaunch(), [torch.zeros(8, 8, 3, dtype=torch.uint8)], None, _NoLaunch(), saved_as=saved_as)


def test_roundtrip_refuses_host_and_malformed_images():
    ok = torch.zeros(1, 8, 8, 3, dtype=torch.uint8)
    with pytest.raises(ValueError, match="CUDA"):
        jpeg.roundtrip_u8(ok)
    with pytest.raises(TypeError):
        jpeg.roundtrip_u8(ok.float())
    with pytest.raises(ValueError, match="quality"):
        jpeg.roundtrip_u8(ok, 0)
    for bad in (ok[0], ok[..., :2], ok.unsqueeze(0)):
        with pytest.raises(ValueError, match="RGB"):
            jpeg.roundtrip_u8(bad)


def test_scratch_bytes():
    assert jpeg.scratch_bytes(1, 1, 1) == 16 * 16 * 3 // 2
    assert jpeg.scratch_bytes(3, 85, 85) == 3 * 96 * 96 * 3 // 2
    assert jpeg.scratch_bytes(2, 255, 257) == 2 * 256 * 272 * 3 // 2
