"""GPU model-level parity at model widths other than 512 and attention widths apart from the model's: the engine against the
reference's outputs in tests/golden/widths.pt (oracle/make_golden_widths.py).  Bars as in test_gpu_model: code indices
bit-exact and pixels (decoding the fixture's codes) within 1e-3 in fp32, 3xTF32 and f16x3; the VAE latent within the
existing VAE goldens' 1e-4.  f16x1 against its numerics model (tests/f16x1_model.py).  Also: packed batches and CUDA graph
replays equal the solo / eager calls bit for bit, and the widths the kernels cannot run are refused, naming the flag,
before any launch."""
import os

import pytest
import torch

import omnitokenizer_b200 as ob
from omnitokenizer_b200 import _cabi
from oracle import omni_oracle as oo
from oracle import weights as W
from tests.f16x1_model import mm_f16x1, provable_near_tie
from tests.util import GOLDEN, check_sub, flags_namespace, flags_setup

pytestmark = pytest.mark.gpu
PIX_TOL = 1e-3
VQ_ROWS = ["w256_h8", "w256_h4", "w512_h4", "w768_h12", "w1024_h16"]


def _math_modes():
    return [m for m in os.environ.get("OMT_TEST_MATH", "fp32,3xtf32,f16x3").split(",") if m]


def widths_golden():
    return torch.load(os.path.join(GOLDEN, "widths.pt"), weights_only=False)


def _model(row, sd, cuda, math, monkeypatch):
    monkeypatch.setenv("OMT_MATH", math)
    m = ob.OmniTokenizer_VQGAN(flags_namespace(row))
    res = m.load_state_dict(sd, strict=False)
    assert not res.missing_keys and not res.unexpected_keys
    m.codebook._need_init = False
    return m.to(cuda).eval()


@pytest.mark.parametrize("math", _math_modes())
@pytest.mark.parametrize("name", VQ_ROWS)
def test_widths_match_golden(cuda, name, math, monkeypatch):
    row = widths_golden()[name]
    cfg, sd, xs = flags_setup(row)
    m = _model(row, sd, cuda, math, monkeypatch)
    eng = m.engine()
    assert (eng.C, eng.A) == (cfg.embedding_dim, cfg.heads * 64)
    for x, r in zip(xs, row["inputs"]):
        is_image = x.ndim == 4
        want = r["idx"].long()
        emb, idx = m.encode(x.to(cuda), is_image, include_embeddings=True)
        mism = int((idx.cpu() != want).sum())
        assert mism == 0, f"{name} {tuple(x.shape)} [{math}]: {mism}/{idx.numel()} code indices differ from the reference"
        check_sub(r["emb"], emb, 1e-5, f"{name} embeddings")
        rec = m.decode(want.to(cuda), is_image)
        err = check_sub(r["rec"], rec, PIX_TOL, f"{name} {tuple(x.shape)} [{math}] reconstruction")
        print(f"{name} {tuple(x.shape)} [{math}]: idx mismatches 0/{idx.numel()}, max |dpixel| {err:.2e}")


@pytest.mark.parametrize("math", _math_modes())
def test_vae_width_matches_golden(cuda, math, monkeypatch):
    row = widths_golden()["w768_vae"]
    cfg, sd, xs = flags_setup(row)
    m = _model(row, sd, cuda, math, monkeypatch)
    x, r = xs[0], row["inputs"][0]
    _orig = torch.randn
    try:       # the reference draws the noise from the global CPU RNG (vae.py:16); inject the recorded draw
        torch.randn = lambda *a, **k: r["noise"].clone()
        z = m.encode(x.to(cuda), False)
    finally:
        torch.randn = _orig
    zerr = check_sub(r["z"], z, 1e-4, "vae latent")
    rec = m.decode(z.permute(0, 2, 3, 4, 1), False)
    err = check_sub(r["rec"], rec, PIX_TOL, "vae reconstruction")
    print(f"w768_vae [{math}]: max |dz| {zerr:.2e}, max |dpixel| {err:.2e}")


@pytest.mark.parametrize("name", VQ_ROWS)
def test_widths_f16x1_within_model_bounds(cuda, name, monkeypatch):
    """f16x1: every flipped code is a provable near-tie (DESIGN.md section 4); pixels from the fixture's codes within 3 x the
    numerics model's error and at most 5e-3."""
    row = widths_golden()[name]
    cfg, sd, xs = flags_setup(row)
    m = _model(row, sd, cuda, "f16x1", monkeypatch)
    eng = m.engine()
    assert eng.h1
    for x, r in zip(xs, row["inputs"]):
        is_image = x.ndim == 4
        ws, _ = eng.encode((x.unsqueeze(2) if is_image else x).to(cuda), "vq")
        idx = ws.idx[: ws.M].cpu()
        z_gpu = eng.z_view(ws).cpu().clone()
        ref = r["idx"].long().reshape(-1)
        flipped = (idx != ref).nonzero().flatten()
        with torch.no_grad():
            h, _ = oo.encoder(sd, cfg, x)
            z = h.reshape(-1, h.shape[-1])
            z = z / z.norm(dim=1, keepdim=True).clamp_min(1e-12)
        if len(flipped):
            ok = provable_near_tie(z[flipped], z_gpu[flipped], sd["codebook.embeddings"], ref[flipped], idx[flipped])
            assert ok.all(), f"{name}: flipped codes that are not near-ties: {flipped[~ok].tolist()}"
        rec = m.decode(r["idx"].long().to(cuda), is_image)
        err = check_sub(r["rec"], rec, 5e-3, f"{name} {tuple(x.shape)} [f16x1] reconstruction")
        with monkeypatch.context() as mp:
            mp.setattr(oo, "MATMUL_MODEL", mm_f16x1)
            with torch.no_grad():
                model_err = check_sub(r["rec"], oo.decode(sd, cfg, r["idx"].long(), is_image), 1.0, "model")
        print(f"{name} {tuple(x.shape)} [f16x1]: flips {len(flipped)}/{ref.numel()}, max |dpx| {err:.2e} "
              f"(model {model_err:.2e})")
        assert err <= 3 * model_err, f"max |dpx| {err:.2e} > 3 x the model's {model_err:.2e}"


@pytest.mark.parametrize("math", _math_modes() + ["f16x1"])
@pytest.mark.parametrize("name", ["w256_h8", "w768_h12"])
def test_widths_mixed_batch_equals_solo_calls(cuda, name, math, monkeypatch):
    """A row's clip and a 1-frame image in one packed pass equal the two solo calls bit for bit, encode and decode."""
    row = widths_golden()[name]
    cfg, sd, xs = flags_setup(row)
    m = _model(row, sd, cuda, math, monkeypatch)
    clip = xs[0][0].to(cuda)
    img = W.synthetic_input(clip.shape[:1] + clip.shape[2:], 3999).to(cuda)
    got = m.encode_batch([clip, img])
    solo_clip, solo_img = m.encode(clip[None], False)[0], m.encode(img[None], True)[0, 0]
    assert torch.equal(got[0], solo_clip) and torch.equal(got[1], solo_img)
    rec = m.decode_batch([solo_clip, solo_img])
    assert torch.equal(rec[0], m.decode(solo_clip[None], False)[0])
    assert torch.equal(rec[1], m.decode(solo_img.reshape(1, -1), True)[0])


@pytest.mark.parametrize("math", ["f16x3", "f16x1", "3xtf32"])
@pytest.mark.parametrize("name", ["w512_h4", "w1024_h16", "w256_h4"])
def test_widths_graph_replay_equals_eager(cuda, name, math, monkeypatch):
    """The first call of a shape runs eagerly, the second captures a CUDA graph and replays it, the third replays it."""
    monkeypatch.setenv("OMT_CUDA_GRAPH", "1")
    row = widths_golden()[name]
    cfg, sd, xs = flags_setup(row)
    m = _model(row, sd, cuda, math, monkeypatch)
    x = xs[0].to(cuda)
    codes = [m.encode(x, False) for _ in range(3)]
    recs = [m.decode(codes[0], False) for _ in range(3)]
    ws = next(iter(m.engine()._ws.values()))
    for slot in ("encode", "decode"):
        assert any(isinstance(g, tuple) for g in ws.graphs_of(slot).values()), f"no {slot} graph was captured"
    for c in codes[1:]:
        assert torch.equal(c, codes[0])
    for r in recs[1:]:
        assert torch.equal(r, recs[0])


# flags on top of the canonical ones (enc_block ttww), and the flag the refusal must name
REJECTED = [
    (["--dim_head", "32"], "dim_head"),
    (["--heads", "7"], "heads"),
    (["--heads", "18"], "heads"),
    (["--embedding_dim", "384"], "embedding_dim"),
    (["--embedding_dim", "1280"], "embedding_dim"),
    (["--embedding_dim", "256"], "heads"),             # ttww with C / heads = 32
    (["--embedding_dim", "1024", "--heads", "8"], "heads"),    # ttww with C / heads = 128
]


@pytest.mark.parametrize("math", _math_modes() + ["f16x1"])
@pytest.mark.parametrize("argv,flag", REJECTED, ids=["dim_head32", "heads7", "heads18", "C384", "C1280", "C256-ttww",
                                                     "C1024-h8-ttww"])
def test_unsupported_widths_are_rejected_before_any_launch(cuda, argv, flag, math, monkeypatch):
    monkeypatch.setenv("OMT_MATH", math)
    m = ob.OmniTokenizer_VQGAN(ob.canonical_args(argv)).to(cuda).eval()
    m.codebook._need_init = False
    n0 = _cabi.launch_count
    with pytest.raises(NotImplementedError, match="--" + flag):
        m.encode(torch.zeros(1, 3, 5, 64, 64, device=cuda), False)
    with pytest.raises(NotImplementedError, match="--" + flag):
        m.decode(torch.zeros(1, 2, 8, 8, dtype=torch.int64, device=cuda), False)
    assert _cabi.launch_count == n0
