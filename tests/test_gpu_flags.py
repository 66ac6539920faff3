"""GPU model-level parity on architecture flags other than the canonical ones: the engine against the reference's outputs in
tests/golden/flags.pt (oracle/make_golden_flags.py) -- causal and non-causal temporal blocks, rel and rope positions, an old
checkpoint's back-filled Namespace, window blocks in the decoder, other block orders and depths, temporal patch 2, other
FF widths, no l2 code.  Bars as in test_gpu_model: code indices bit-exact, pixels within 1e-3 abs.  Decoding the fixture's
codes (not the engine's own) keeps encoder and decoder faults apart.  Also: what the kernels cannot run is rejected, naming the
flag, before any launch."""
import os

import pytest
import torch

import omnitokenizer_b200 as ob
from omnitokenizer_b200 import _cabi
from oracle import weights as W
from tests.util import GOLDEN, check_sub, flags_namespace, flags_setup

pytestmark = pytest.mark.gpu
PIX_TOL = 1e-3
ROWS = ["backfill", "stage1", "attn_causal_only", "peg_causal_only", "blocks", "ff2", "ff3", "nol2"]
# rows whose video goes through encode_batch / decode_batch next to an image: the varlen PEG and temporal attention entry
# points with each causal flag on its own and with neither
BATCH_ROWS = ["backfill", "attn_causal_only", "peg_causal_only"]


def _math_modes():
    return [m for m in os.environ.get("OMT_TEST_MATH", "fp32,3xtf32,f16x3").split(",") if m]


def flags_golden():
    return torch.load(os.path.join(GOLDEN, "flags.pt"), weights_only=False)


def _model(row, sd, cuda, math, monkeypatch):
    monkeypatch.setenv("OMT_MATH", math)
    m = ob.OmniTokenizer_VQGAN(flags_namespace(row))
    res = m.load_state_dict(sd, strict=False)
    assert not res.missing_keys and not res.unexpected_keys, (res.missing_keys[:3], res.unexpected_keys[:3])
    m.codebook._need_init = False
    return m.to(cuda).eval()


@pytest.mark.parametrize("math", _math_modes())
@pytest.mark.parametrize("name", ROWS)
def test_flags_match_golden(cuda, name, math, monkeypatch):
    row = flags_golden()[name]
    cfg, sd, xs = flags_setup(row)
    m = _model(row, sd, cuda, math, monkeypatch)
    for x, r in zip(xs, row["inputs"]):
        is_image = x.ndim == 4
        want = r["idx"].long()
        emb, idx = m.encode(x.to(cuda), is_image, include_embeddings=True)
        assert idx.dtype == torch.int64 and tuple(idx.shape) == tuple(want.shape)
        mism = int((idx.cpu() != want).sum())
        assert mism == 0, f"{name} {tuple(x.shape)} [{math}]: {mism}/{idx.numel()} code indices differ from the reference"
        assert (emb.cpu() - r["emb"]).abs().max().item() <= 1e-5
        rec = m.decode(want.to(cuda), is_image)
        err = check_sub(r["rec"], rec, PIX_TOL, f"{name} {tuple(x.shape)} [{math}] reconstruction")
        print(f"{name} {tuple(x.shape)} [{math}]: idx mismatches 0/{idx.numel()}, max |dpixel| {err:.2e}")


@pytest.mark.parametrize("math", _math_modes())
@pytest.mark.parametrize("name", BATCH_ROWS)
def test_flags_mixed_batch_equals_solo_calls(cuda, name, math, monkeypatch):
    """A row's clip and a 1-frame image in one packed pass equal the two solo calls bit for bit, encode and decode."""
    row = flags_golden()[name]
    cfg, sd, xs = flags_setup(row)
    m = _model(row, sd, cuda, math, monkeypatch)
    clip = xs[0][0].to(cuda)
    img = W.synthetic_input(clip.shape[:1] + clip.shape[2:], 2999).to(cuda)
    got = m.encode_batch([clip, img])
    solo_clip, solo_img = m.encode(clip[None], False)[0], m.encode(img[None], True)[0, 0]
    assert torch.equal(got[0], solo_clip) and torch.equal(got[1], solo_img)
    assert torch.equal(solo_clip.cpu(), row["inputs"][0]["idx"].long()[0])
    rec = m.decode_batch([solo_clip, solo_img])
    assert torch.equal(rec[0], m.decode(solo_clip[None], False)[0])
    assert torch.equal(rec[1], m.decode(solo_img.reshape(1, -1), True)[0])


# flag the message names, its value (on top of the canonical flags), input shape, math modes the kernels cannot run it in
REJECTED = [
    ("twod_window_size", 4, (1, 3, 5, 64, 64), ("fp32", "3xtf32", "f16x3")),     # window blocks: enc_block ttww
    ("patch_size", 16, (1, 3, 5, 128, 128), ("fp32", "3xtf32", "f16x3")),        # patch K 3 * 4 * 16^2 = 3072 > 1024
    ("patch_size", 4, (1, 3, 5, 64, 64), ("3xtf32", "f16x3")),                   # patch K 48: not a whole k-block
    ("codebook_dim", 16, (1, 3, 5, 64, 64), ("fp32", "3xtf32", "f16x3")),        # without --use_vae
]


@pytest.mark.parametrize("math", _math_modes())
@pytest.mark.parametrize("flag,value,shape,modes", REJECTED, ids=[f"{c[0]}-{c[1]}" for c in REJECTED])
def test_unsupported_flags_are_rejected_before_any_launch(cuda, flag, value, shape, modes, math, monkeypatch):
    if math not in modes:
        pytest.skip(f"{math} runs this configuration")
    monkeypatch.setenv("OMT_MATH", math)
    m = ob.OmniTokenizer_VQGAN(ob.canonical_args(["--" + flag, str(value)])).to(cuda).eval()
    m.codebook._need_init = False
    x = torch.zeros(shape, device=cuda)
    n0 = _cabi.launch_count
    with pytest.raises((NotImplementedError, ValueError), match=flag):
        m.encode(x, False)
    assert _cabi.launch_count == n0
    if (flag, value) != ("patch_size", 16):         # patch 16 decodes: only the encoder's patch gather is limited
        h = shape[-1] // (value if flag == "patch_size" else 8)
        with pytest.raises((NotImplementedError, ValueError), match=flag):
            m.decode(torch.zeros(1, 2, h, h, dtype=torch.int64, device=cuda), False)
        assert _cabi.launch_count == n0
