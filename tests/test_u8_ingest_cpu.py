"""CPU checks of the uint8 input side (encode_u8 / forward_u8 and the consumers' *_u8 functions): the byte tables against the
reference pipelines' own outputs (tests/golden/u8_norm.pt, oracle/make_golden_u8.py), the VideoNorm restatement, the host
fallbacks of the consumer functions and argument validation."""
import os

import pytest
import torch

from omnitokenizer_b200 import consumers as C
from omnitokenizer_b200 import layout as L
from oracle import omni_oracle as oo
from oracle import weights as W
from oracle.u8_norm import video_norm
from tests.test_consumers_cpu import _OracleBacked

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "u8_norm.pt")
PRESETS = {"video_norm": C.VIDEO_NORM, "image_norm": C.IMAGE_NORM, "dit_norm": C.DIT_NORM, "latte_norm": C.LATTE_NORM}


@pytest.fixture(scope="module")
def fx():
    return torch.load(GOLDEN, weights_only=False)


def _table_from_fixture(clip, out_tchw):
    """[C, 256] byte -> value map read off a reference output; every byte occurs in every channel of the clip."""
    T, H, W, Cn = clip.shape
    tab = torch.full((Cn, 256), float("nan"))
    for c in range(Cn):
        tab[c, clip[..., c].reshape(-1).long()] = out_tchw[:, c].reshape(-1)
    return tab


@pytest.mark.parametrize("name", sorted(PRESETS))
def test_tables_equal_reference_pipelines(fx, name):
    clip = fx["clip"]
    for c in range(3):
        assert torch.equal(clip[..., c].reshape(-1).unique(), torch.arange(256, dtype=torch.uint8))
    ref = fx[name].permute(1, 0, 2, 3) if name == "video_norm" else fx[name]          # -> (T, C, H, W)
    tab = L.u8_norm_table(PRESETS[name], 3)
    assert tab.dtype == torch.float32 and tuple(tab.shape) == ((2 if name == "video_norm" else 1), 3, 256)
    assert torch.equal(tab[0], _table_from_fixture(clip, ref))
    if name == "video_norm":                                   # table 1: the undivided map of clips with max <= 1
        for mx in (0, 1):
            q = fx["quirk"][mx]
            got = fx["video_norm_quirk"][mx].permute(1, 0, 2, 3)
            for c in range(3):
                u = q[..., c].reshape(-1).long()
                assert torch.equal(tab[1, c, u], got[:, c].reshape(-1))
        want1 = (torch.arange(256).float().view(1, 256) - 0.5) / 1.0
        assert torch.equal(tab[1], want1.expand(3, 256))


def test_video_norm_restatement_matches_reference(fx):
    assert torch.equal(video_norm(fx["clip"][None])[0], fx["video_norm"])
    for mx, q in fx["quirk"].items():
        assert int(q.max()) == mx
        assert torch.equal(video_norm(q[None])[0], fx["video_norm_quirk"][mx])
    # the host table path agrees, per sample, on a batch mixing the quirk clips with a full one
    batch = torch.stack([fx["clip"], fx["quirk"][0], fx["quirk"][1], fx["quirk"][2]])
    assert torch.equal(L.u8_normalize(batch, C.VIDEO_NORM), video_norm(batch))


def test_reciprocal_division_is_not_the_pipeline():
    """Why the values come from a host table: multiplying by 1/255 (what a CUDA division by a scalar does) is not u / 255."""
    u = torch.arange(256).float()
    assert int((u / 255.0 != u * (1.0 / 255.0)).sum()) > 0


def _frames(shape, seed):
    return torch.randint(0, 256, shape, generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)


def test_consumer_fallbacks_equal_fp32_counterparts():
    cfg = oo.Config(resolution=64)
    sd = W.make_state_dict(cfg, 22)
    m = _OracleBacked(cfg, sd)
    f = _frames((1, 5, 64, 64, 3), 3)
    x = video_norm(f)
    for n in (0, 2):
        got = C.encode_to_z_u8(m, f, False, n)
        want = C.encode_to_z(m, x, False, n)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    total, total_ref = torch.zeros(8192), torch.zeros(8192)
    out, vq = C.eval_step_u8(m, f, total)
    _, frames_ref, vq_ref = C.eval_step(m, x, total_ref)
    assert torch.equal(out, frames_ref) and torch.equal(vq["encodings"], vq_ref["encodings"]) and torch.equal(total, total_ref)

    cfg = oo.Config(use_vae=True, resolution=64)
    sd = W.make_state_dict(cfg, 23)
    img = _frames((2, 64, 64, 3), 4)
    noise = torch.randn((2, 8, 1, 8, 8), generator=torch.Generator().manual_seed(3))
    m = _OracleBacked(cfg, sd, noise)
    xi = L.u8_normalize(img.unsqueeze(1), C.DIT_NORM).squeeze(2)
    assert torch.equal(C.dit_encode_latents_u8(m, img), C.dit_encode_latents(m, xi))
    clips = _frames((1, 5, 64, 64, 3), 5)
    noise = torch.randn((1, 8, 2, 8, 8), generator=torch.Generator().manual_seed(4))
    m = _OracleBacked(cfg, sd, noise)
    xv = L.u8_normalize(clips, C.LATTE_NORM).permute(0, 2, 1, 3, 4)           # 'b f c h w', the Latte loader's layout
    assert torch.equal(C.latte_encode_latents_u8(m, clips), C.latte_encode_latents(m, xv))


def test_argument_validation():
    cfg = oo.Config(resolution=64)
    m = _OracleBacked(cfg, W.make_state_dict(cfg, 22))
    with pytest.raises(TypeError):
        C.encode_to_z_u8(m, torch.zeros(1, 5, 64, 64, 3), False)              # fp32, not uint8
    with pytest.raises(ValueError):
        C.encode_to_z_u8(m, torch.zeros(1, 64, 64, 3, dtype=torch.uint8), False)   # a video needs 5 dimensions
    with pytest.raises(ValueError):
        C.encode_to_z_u8(m, torch.zeros(1, 5, 64, 64, 4, dtype=torch.uint8), False)   # 4 channels, 3-channel preset
    with pytest.raises(TypeError):
        C.eval_step_u8(m, torch.zeros(1, 5, 64, 64, 3, dtype=torch.int16))
    with pytest.raises(ValueError):
        L.u8_norm_table(C.DIT_NORM, 1)


def test_module_rejects_bad_frames_before_launch():
    """OmniTokenizer_VQGAN validates uint8 input on the host (no device needed to get the error)."""
    import omnitokenizer_b200 as ob
    m = ob.OmniTokenizer_VQGAN(ob.canonical_args())
    with pytest.raises(TypeError):
        m.encode_u8(torch.zeros(1, 5, 64, 64, 3), False)
    with pytest.raises(ValueError):
        m.encode_u8(torch.zeros(1, 5, 64, 64, 4, dtype=torch.uint8), False)
    with pytest.raises(ValueError):
        m.encode_u8(torch.zeros(1, 5, 64, 64, 3, dtype=torch.uint8), True)
    with pytest.raises(TypeError):
        m.forward_u8(torch.zeros(1, 5, 64, 64, 3, dtype=torch.float32))
    m.resolution_scale = [0.5]
    with pytest.raises(NotImplementedError):
        m.forward_u8(torch.zeros(1, 5, 64, 64, 3, dtype=torch.uint8))
