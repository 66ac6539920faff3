"""GPU checks of the uint8 input side: omt_patchify_ln_u8 against omt_patchify_ln on the table-mapped fp32 video, VideoNorm's
per-clip table select, and encode_u8 / forward_u8 against encode / forward on the pipeline's fp32 input (oracle video_norm)
on every golden configuration.  Every comparison is exact (torch.equal)."""
import os

import pytest
import torch

from omnitokenizer_b200 import _cabi
from omnitokenizer_b200 import consumers as C
from omnitokenizer_b200 import layout as L
from omnitokenizer_b200.engine import default_math
from oracle import omni_oracle as oo
from oracle import weights as W
from oracle.u8_norm import video_norm
from tests.util import GOLDEN_CASES, build_model, golden_setup, load_golden

pytestmark = pytest.mark.gpu
MATHS = [m for m in os.environ.get("OMT_TEST_MATH", "fp32,3xtf32,f16x3").split(",") if m]


def _frames(shape, seed, hi=256):
    return torch.randint(0, hi, shape, generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)


def _materialise(frames, tab, sel):
    """(B,T,H,W,C) bytes -> (B,C,T,H,W) fp32 through table sel[b] (a lookup: exact)."""
    B, C = frames.shape[0], frames.shape[-1]
    x = frames.permute(0, 4, 1, 2, 3).long()
    return tab[sel.long().view(B, 1, 1, 1, 1), torch.arange(C, device=frames.device).view(1, C, 1, 1, 1), x].contiguous()


@pytest.mark.parametrize("B,T,H", [(1, 1, 64), (2, 5, 64), (3, 9, 128), (1, 17, 256)])
def test_patchify_ln_u8_equals_fp32_gather(cuda, B, T, H):
    _cabi.load()
    p, pt, Cin = 8, 4, 3
    g = torch.Generator().manual_seed(B * 100 + T)
    frames = _frames((B, T, H, H, Cin), T + H).to(cuda)
    tab = L.u8_norm_table(C.VIDEO_NORM, Cin).to(cuda)
    sels = [None, torch.tensor([b % 2 for b in range(B)], dtype=torch.int32, device=cuda),
            torch.tensor([(b + 1) % 2 for b in range(B)], dtype=torch.int32, device=cuda)]
    for first in ((1,) if T == 1 else (1, 0)):
        PT = 1 if first else pt
        K = Cin * PT * p * p
        rows = B * (1 if first else (T - 1) // pt) * (H // p) ** 2
        lw = (torch.rand(K, generator=g) + 0.5).to(cuda)
        lb = ((torch.rand(K, generator=g) - 0.5) * 0.2).to(cuda)
        for sel in sels:
            video = _materialise(frames, tab, sel if sel is not None else torch.zeros(B, dtype=torch.int32, device=cuda))
            lut = tab if sel is not None else tab[:1].contiguous()
            for ln in ((lw, lb), (None, None)):
                # fp32 A
                a0 = torch.full((rows, K), float("nan"), device=cuda)
                a1 = torch.full((rows, K), float("nan"), device=cuda)
                _cabi.call("omt_patchify_ln", video, a0, None, None, None, *ln, B, Cin, T, H, H, p, pt, first, 1e-5)
                _cabi.call("omt_patchify_ln_u8", frames, lut, sel, a1, None, None, None, *ln, B, Cin, T, H, H, p, pt, first, 1e-5)
                assert torch.equal(a0, a1)
                # 2^11-scaled planes and row-scaled planes (+ inverse row scales)
                for rs in (False, True):
                    outs = []
                    for _ in range(2):
                        pl = torch.full((2, rows, K), -1, dtype=torch.int16, device=cuda)
                        r = torch.full((rows,), float("nan"), device=cuda) if rs else None
                        outs.append((pl, r))
                    _cabi.call("omt_patchify_ln", video, None, outs[0][0][0], outs[0][0][1], outs[0][1], *ln, B, Cin, T, H, H,
                               p, pt, first, 1e-5)
                    _cabi.call("omt_patchify_ln_u8", frames, lut, sel, None, outs[1][0][0], outs[1][0][1], outs[1][1], *ln, B,
                               Cin, T, H, H, p, pt, first, 1e-5)
                    assert torch.equal(outs[0][0], outs[1][0])
                    if rs:
                        assert torch.equal(outs[0][1], outs[1][1])


def test_u8_norm_select(cuda):
    _cabi.load()
    clips = [_frames((5, 64, 64, 3), 1, hi=1), _frames((5, 64, 64, 3), 2, hi=2), _frames((5, 64, 64, 3), 3, hi=3),
             _frames((5, 64, 64, 3), 4)]
    clips[1][4, 63, 63, 2] = 1
    clips[2][0, 0, 0, 0] = 2
    clips[3][2, 10, 10, 1] = 255
    frames = torch.stack(clips).to(cuda)
    assert [int(c.max()) for c in clips] == [0, 1, 2, 255]
    sel = torch.full((4,), 7, dtype=torch.int32, device=cuda)
    _cabi.call("omt_u8_norm_select", frames, 4, frames[0].numel(), sel)
    assert sel.tolist() == [1, 1, 0, 0]
    # a single byte of 2 at the very end of a sample, and an unaligned per-sample size (byte path)
    f = torch.zeros((2, 1, 1, 5, 3), dtype=torch.uint8, device=cuda)
    f[1, 0, 0, 4, 2] = 2
    _cabi.call("omt_u8_norm_select", f, 2, 15, sel)
    assert sel[:2].tolist() == [1, 0]


def _usage_state(m):
    return m.codebook.codebook_usage.clone(), m.codebook.call_cnt


def _set_usage_state(m, st):
    m.codebook.codebook_usage.data = st[0].clone()
    m.codebook.call_cnt = st[1]


def _golden_frames(fx, seed):
    shape = tuple(fx["shape"])
    if len(shape) == 4:
        B, Cn, H, W_ = shape
        return _frames((B, H, W_, Cn), seed)
    B, Cn, T, H, W_ = shape
    return _frames((B, T, H, W_, Cn), seed)


def _eq(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_eq(a[k], b[k]) for k in a)
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(_eq(x, y) for x, y in zip(a, b))
    if a is None or b is None:
        return a is b
    return torch.equal(a, b)


@pytest.mark.parametrize("math", MATHS)
@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_encode_u8_and_forward_u8_equal_fp32_path(cuda, name, math):
    fx = load_golden(name)
    cfg, sd, _ = golden_setup(fx)
    m = build_model(cfg, sd, cuda, math)
    frames = _golden_frames(fx, 17)
    is_image = frames.ndim == 4
    x = video_norm(frames.unsqueeze(1) if is_image else frames)
    x = (x.squeeze(2) if is_image else x).to(cuda)
    fr = frames.to(cuda)
    st0 = _usage_state(m)
    for emb in ((False, True) if not cfg.use_vae else (False,)):
        _set_usage_state(m, st0)
        torch.manual_seed(11)
        want = m.encode(x, is_image, include_embeddings=emb)
        st_want, rng_want = _usage_state(m), torch.get_rng_state()
        _set_usage_state(m, st0)
        torch.manual_seed(11)
        got = m.encode_u8(fr, is_image, include_embeddings=emb)
        assert _eq(got, want), f"{name} [{math}] encode_u8 != encode (include_embeddings={emb})"
        assert _eq(_usage_state(m)[0], st_want[0]) and _usage_state(m)[1] == st_want[1]
        assert torch.equal(torch.get_rng_state(), rng_want)
    # forward(log_image=True) + the eval script's byte conversion
    _set_usage_state(m, st0)
    torch.manual_seed(12)
    _, _, _, xr, vq = m(x, log_image=True)
    want_u8 = C._to_u8(xr.unsqueeze(2) if is_image else xr, C.EVAL_U8)
    st_want, rng_want = _usage_state(m), torch.get_rng_state()
    _set_usage_state(m, st0)
    torch.manual_seed(12)
    got_u8, vq_u8 = m.forward_u8(fr)
    assert torch.equal(got_u8, want_u8) and _eq(vq_u8, vq)
    assert _eq(_usage_state(m)[0], st_want[0]) and _usage_state(m)[1] == st_want[1]
    assert torch.equal(torch.get_rng_state(), rng_want)


def test_encode_u8_slot_graphs_interleave_with_encode_slot(cuda):
    """Same shape through encode and encode_u8: each call path runs eagerly, then captures, then replays a graph."""
    cfg = oo.Config(resolution=64)
    m = build_model(cfg, W.make_state_dict(cfg, 2), cuda, default_math())
    frames = [_frames((2, 5, 64, 64, 3), 30 + i) for i in range(3)]
    frames[1][0] = frames[1][0] % 2                 # a clip VideoNorm leaves undivided
    outs = []
    for f in frames:
        a = m.encode_u8(f.to(cuda), False)
        b = m.encode(video_norm(f).to(cuda), False)
        outs.append((a, b))
    for a, b in outs:
        assert torch.equal(a, b)
    assert not torch.equal(outs[0][0], outs[2][0])
    ws = next(iter(m.engine()._ws.values()))
    assert ws.graphs_of("encode") and ws.graphs_of("encode_u8") and all(not isinstance(v, str) for v in ws.graphs.values())


def test_fullsize_cfg3_codes(cuda):
    """One cfg-3 batch (8 x 17 x 256^2 uint8 frames): the codes equal the fp32 path's."""
    cfg = oo.Config()
    m = build_model(cfg, W.make_state_dict(cfg, 0), cuda, default_math())
    frames = _frames((8, 17, 256, 256, 3), 99)
    a = m.encode_u8(frames.to(cuda), False)
    b = m.encode(video_norm(frames).to(cuda), False)
    assert torch.equal(a, b)


def test_u8_errors(cuda):
    cfg = oo.Config(resolution=64)
    m = build_model(cfg, W.make_state_dict(cfg, 0), cuda, "fp32")
    with pytest.raises(TypeError):
        m.encode_u8(torch.zeros(1, 5, 64, 64, 3, device=cuda), False)
    with pytest.raises(ValueError):
        m.encode_u8(torch.zeros(1, 5, 64, 64, 1, dtype=torch.uint8, device=cuda), False)
    with pytest.raises(AssertionError, match="divisible by temporal patch size"):
        m.encode_u8(torch.zeros(1, 6, 64, 64, 3, dtype=torch.uint8, device=cuda), False)
    m.resolution_scale = [0.5, 1.0]
    with pytest.raises(NotImplementedError):
        m.forward_u8(torch.zeros(1, 5, 64, 64, 3, dtype=torch.uint8, device=cuda))
    # the C entry point checks its arguments too
    f = torch.zeros(1, 6, 64, 64, 3, dtype=torch.uint8, device=cuda)
    lut = L.u8_norm_table(C.DIT_NORM, 3).to(cuda)
    A = torch.empty(16 * 768, device=cuda)
    with pytest.raises(RuntimeError, match=r"\(T-1\)"):
        _cabi.call("omt_patchify_ln_u8", f, lut, None, A, None, None, None, None, None, 1, 3, 6, 64, 64, 8, 4, 0, 1e-5)
    with pytest.raises(RuntimeError, match="Cin"):
        _cabi.call("omt_patchify_ln_u8", f, lut, None, A, None, None, None, None, None, 1, 5, 5, 64, 64, 8, 4, 0, 1e-5)
    with pytest.raises(RuntimeError, match="null"):
        _cabi.call("omt_patchify_ln_u8", f, None, None, A, None, None, None, None, None, 1, 3, 5, 64, 64, 8, 4, 0, 1e-5)
    # B == 0 follows encode's empty result
    m.resolution_scale = None
    e = m.encode_u8(torch.zeros(0, 5, 64, 64, 3, dtype=torch.uint8, device=cuda), False)
    assert tuple(e.shape) == (0, 2, 8, 8) and e.dtype == torch.int64
