"""Packed batches of different lengths: the layout-table kernels (omt_peg_volume_varlen, omt_attn_temporal_varlen) against
per-sample launches of the uniform entry points, and OmniTokenizer_VQGAN.encode_batch / decode_batch / decode_u8_batch
against the sequential per-element calls -- bit for bit, side effects included."""
import os

import pytest
import torch

from oracle import omni_oracle as oo
from oracle import weights as W
from tests.util import build_model, check_sub, golden_setup, load_golden

pytestmark = pytest.mark.gpu
PIX_TOL = 1e-3
# every T' from 1 to 17, unsorted, with repeats
LENGTHS = [5, 1, 17, 3, 5, 2, 9, 1, 16, 4, 6, 7, 8, 10, 11, 12, 13, 14, 15, 3]


def _cabi():
    from omnitokenizer_b200 import _cabi as c
    c.load()
    return c


def _t_off(lengths, cuda):
    t = torch.tensor([0] + lengths, dtype=torch.int32).cumsum(0).to(torch.int32)
    return t, t.to(cuda)


def _rand(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g) * scale


# ---------------------------------------------------------------- kernels

def _temporal(qkv, o, op, lengths, N, causal, cuda, varlen=True):
    """Temporal attention over the packed qkv [M, 1536]: one varlen launch, or one uniform launch per sample."""
    c = _cabi()
    p, M = qkv.data_ptr(), qkv.shape[0]
    out = (o, None, None) if op is None else (None, op[0], op[1])
    if varlen:
        th, td = _t_off(lengths, cuda)
        c.call("omt_attn_temporal_varlen", p, 1536, p + 2048, 1536, p + 4096, 1536, *out, 512, th, td, len(lengths), M, N, 8,
               8.0, causal)
        return
    f = 0
    for t in lengths:
        r = f * N
        po = (o.data_ptr() + r * 512 * 4, None, None) if op is None else \
            (None, op[0].data_ptr() + r * 512 * 2, op[1].data_ptr() + r * 512 * 2)
        c.call("omt_attn_temporal", p + r * 1536 * 4, 1536, p + r * 1536 * 4 + 2048, 1536, p + r * 1536 * 4 + 4096, 1536,
               *po, 512, 1, t, N, 8, 8.0, causal)
        f += t


@pytest.mark.parametrize("planes", [False, True])
@pytest.mark.parametrize("causal", [1, 0])
def test_temporal_varlen_equals_per_sample(cuda, causal, planes):
    N = 64
    M = sum(LENGTHS) * N
    qkv = (_rand((M, 1536), 50) * 0.5).to(cuda)
    outs = []
    for varlen in (True, False):
        o = torch.full((M, 512), float("nan"), device=cuda)
        op = (torch.zeros(M, 512, dtype=torch.int16, device=cuda), torch.zeros(M, 512, dtype=torch.int16, device=cuda)) if planes else None
        _temporal(qkv, o, op, LENGTHS, N, causal, cuda, varlen)
        torch.cuda.synchronize()
        outs.append(torch.cat(op) if planes else o)
    assert torch.equal(outs[0], outs[1])
    if not planes:
        assert bool(torch.isfinite(outs[0]).all())


def _peg(x, y, wt, bias, lengths, h, w, temporal, causal, cuda, varlen=True):
    c = _cabi()
    C = x.shape[1]
    if varlen:
        th, td = _t_off(lengths, cuda)
        c.call("omt_peg_volume_varlen", x, y, wt, bias, th, td, len(lengths), x.shape[0], h, w, C, int(temporal), int(causal))
        return
    f = 0
    for t in lengths:
        r = f * h * w
        c.call("omt_peg_volume", x.data_ptr() + r * C * 4, y.data_ptr() + r * C * 4, wt, bias, 1, t, h, w, C, int(temporal),
               int(causal))
        f += t


@pytest.mark.parametrize("pk", [4, 3])
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("temporal", [False, True])
def test_peg_varlen_equals_per_sample(cuda, temporal, causal, pk):
    c = _cabi()
    c.set_option("peg_kernel", pk)
    h = w = 8
    C = 64
    M = sum(LENGTHS) * h * w
    x = _rand((M, C), 23).to(cuda)
    wt, bias = _rand((27, C), 24, 0.3).to(cuda), _rand((C,), 25, 0.1).to(cuda)
    outs = []
    for varlen in (True, False):
        y = torch.full((M, C), float("nan"), device=cuda)
        _peg(x, y, wt, bias, LENGTHS, h, w, temporal, causal, cuda, varlen)
        torch.cuda.synchronize()
        outs.append(y)
    assert torch.equal(outs[0], outs[1])
    assert bool(torch.isfinite(outs[0]).all())
    # and the per-sample results are the oracle's PEG of each sample alone
    f = 0
    for t in LENGTHS[:3]:
        xs = x[f * h * w:(f + t) * h * w].cpu().view(1, t, h * w, C)
        want = oo.peg(xs, wt.cpu().t().reshape(C, 1, 3, 3, 3), bias.cpu(), (h, w), temporal, causal) + xs
        assert (outs[0][f * h * w:(f + t) * h * w].cpu().view_as(want) - want).abs().max().item() < 1e-5
        f += t


@pytest.mark.parametrize("kind", ["peg_spatial", "peg_temporal", "attn"])
def test_neighbours_never_leak(cuda, kind):
    """Poisoning every other sample's rows (NaN, huge values) leaves sample b's output bit-identical and finite."""
    h = w = 8
    N = h * w
    lengths = [3, 5, 1, 5, 2]
    M = sum(lengths) * N
    C = 1536 if kind == "attn" else 64
    clean = (_rand((M, C), 60) * 0.5).to(cuda)
    wt, bias = _rand((27, 64), 61, 0.3).to(cuda), _rand((64,), 62, 0.1).to(cuda)

    def run(x):
        if kind == "attn":
            o = torch.empty(M, 512, device=cuda)
            _temporal(x, o, None, lengths, N, 1, cuda)
        else:
            o = torch.empty(M, 64, device=cuda)
            _peg(x, o, wt, bias, lengths, h, w, kind == "peg_temporal", True, cuda)
        torch.cuda.synchronize()
        return o

    ref = run(clean)
    offs = [0]
    for t in lengths:
        offs.append(offs[-1] + t)
    for b in range(len(lengths)):
        lo, hi = offs[b] * N, offs[b + 1] * N
        for poison in (float("nan"), 3e38):
            x = torch.full_like(clean, poison)
            x[lo:hi] = clean[lo:hi]
            got = run(x)
            assert torch.equal(got[lo:hi], ref[lo:hi]), (b, poison)
            assert bool(torch.isfinite(got[lo:hi]).all())


@pytest.mark.parametrize("entry", ["omt_peg_volume_varlen", "omt_attn_temporal_varlen"])
def test_bad_tables_raise_before_launch(cuda, entry):
    c = _cabi()
    h = w = 8
    N = h * w
    good = [3, 5, 1]
    M = sum(good) * N
    x = _rand((M, 1536), 70).to(cuda)
    bad = {"decreasing": [0, 3, 2, 9], "wrong total": [0, 3, 8, 10], "zero length": [0, 3, 3, 9], "T'=18": [0, 1, 19, 19],
           "first not 0": [1, 4, 9, 10]}
    for what, tab in bad.items():
        th = torch.tensor(tab, dtype=torch.int32)
        td = th.to(cuda)
        sentinel = torch.full((M, 512), 7.0, device=cuda)
        with pytest.raises(RuntimeError, match=entry):
            if entry == "omt_peg_volume_varlen":
                c.call(entry, x[:, :64].contiguous(), sentinel[:, :64], x[:27, :64].contiguous(), x[0, :64].contiguous(),
                       th, td, 3, M, h, w, 64, 1, 1)
            else:
                p = x.data_ptr()
                c.call(entry, p, 1536, p + 2048, 1536, p + 4096, 1536, sentinel, None, None, 512, th, td, 3, M, N, 8, 8.0, 1)
        torch.cuda.synchronize()
        assert bool((sentinel == 7.0).all()), f"{what}: a rejected launch wrote outputs"


# ---------------------------------------------------------------- the model

def _math_modes():
    return [m for m in os.environ.get("OMT_TEST_MATH", "fp32,3xtf32,f16x3").split(",") if m]


def _inputs():
    """Images and clips with T' from 1 to 17 (unsorted, repeats) plus the img64 / vid5x64 golden inputs."""
    img = golden_setup(load_golden("img64"))[2][0]                 # (3, 64, 64)
    vid = golden_setup(load_golden("vid5x64"))[2][0]               # (3, 5, 64, 64)
    xs = [vid, W.synthetic_input((1, 3, 64, 64), 1)[0], img]
    for k, tp in enumerate([3, 1, 17, 2, 5, 9, 4, 3, 6, 7, 8, 10, 11, 12, 13, 14, 15, 16]):
        xs.append(W.synthetic_input((1, 3, 1 + 4 * (tp - 1), 64, 64), 100 + k)[0])
    xs.append(W.synthetic_input((1, 3, 64, 64), 2)[0])
    return xs


def _seq_encode(m, xs, cuda, **kw):
    return [m.encode(x[None].to(cuda), x.ndim == 3, **kw) for x in xs]


@pytest.mark.parametrize("math", _math_modes())
def test_vq_batch_equals_sequential_calls(cuda, math):
    cfg, sd, _ = golden_setup(load_golden("img64"))
    a = build_model(cfg, sd, cuda, math)          # batch calls
    b = build_model(cfg, sd, cuda, math)          # the sequential calls, same weights
    xs = _inputs()
    got = a.encode_batch([x.to(cuda) for x in xs])
    want = _seq_encode(b, xs, cuda)
    assert len(got) == len(xs)
    for x, g, wnt in zip(xs, got, want):
        assert torch.equal(g, wnt[0, 0] if x.ndim == 3 else wnt[0])
    assert a.codebook.call_cnt == b.codebook.call_cnt == len(xs)
    assert torch.equal(a.codebook.codebook_usage, b.codebook.codebook_usage)
    # with embeddings (moves the statistics once more per element, like encode does)
    got_e = a.encode_batch(xs, include_embeddings=True)
    want_e = _seq_encode(b, xs, cuda, include_embeddings=True)
    for x, (ge, gi), (we, wi) in zip(xs, got_e, want_e):
        if x.ndim == 3:
            assert torch.equal(ge, we[0, :, 0]) and torch.equal(gi, wi[0, 0])
        else:
            assert torch.equal(ge, we[0]) and torch.equal(gi, wi[0])
    assert a.codebook.call_cnt == b.codebook.call_cnt == 2 * len(xs)
    assert torch.equal(a.codebook.codebook_usage, b.codebook.codebook_usage)
    # decode / decode_u8 of the returned codes
    rec = a.decode_batch(got)
    rec8 = a.decode_u8_batch(got)
    rec8b = a.decode_u8_batch(got, affine=(255.0, 128.0, 0.0, 255.0, 1.0))
    for x, g, r, r8, r8b in zip(xs, got, rec, rec8, rec8b):
        img = x.ndim == 3
        e = g.reshape(1, 1, *g.shape) if img else g[None]
        assert torch.equal(r, b.decode(e, img)[0])
        assert torch.equal(r8, b.decode_u8(e, img)[0])
        assert torch.equal(r8b, b.decode_u8(e, img, affine=(255.0, 128.0, 0.0, 255.0, 1.0))[0])
    # the golden elements against their fixtures
    for pos, name in ((2, "img64"), (0, "vid5x64")):
        fx = load_golden(name)
        assert torch.equal(got[pos].cpu().reshape(fx["idx"].shape), fx["idx"].long())
        emb = got_e[pos][0]
        check_sub(fx["emb"], emb[None] if name == "vid5x64" else emb[None, :, None], 1e-5, name + " embeddings")
        check_sub(fx["rec"], rec[pos][None], PIX_TOL, name + " reconstruction")


@pytest.mark.parametrize("math", _math_modes())
def test_vae_batch_equals_sequential_calls(cuda, math):
    cfg, sd, _ = golden_setup(load_golden("vae_vid5x64"))
    m = build_model(cfg, sd, cuda, math)
    xs = [W.synthetic_input((1, 3, 9, 64, 64), 7)[0], W.synthetic_input((1, 3, 64, 64), 8)[0],
          W.synthetic_input((1, 3, 5, 64, 64), 9)[0], W.synthetic_input((1, 3, 64, 64), 10)[0],
          W.synthetic_input((1, 3, 1, 64, 64), 11)[0]]
    torch.manual_seed(1234)
    got = m.encode_batch([x.to(cuda) for x in xs])
    state_batch = torch.get_rng_state()
    torch.manual_seed(1234)
    want = _seq_encode(m, xs, cuda)
    assert torch.equal(state_batch, torch.get_rng_state())
    for g, wnt in zip(got, want):
        assert torch.equal(g, wnt[0])
    lat = [g if x.ndim == 3 else g.permute(1, 2, 3, 0) for x, g in zip(xs, got)]       # decode's 't h w c' video form
    rec, rec8 = m.decode_batch(lat), m.decode_u8_batch(lat)
    for x, l, r, r8 in zip(xs, lat, rec, rec8):
        img = x.ndim == 3
        assert torch.equal(r, m.decode(l[None], img)[0])
        assert torch.equal(r8, m.decode_u8(l[None], img)[0])
    # the golden video through a batch: its latents with the recorded noise
    fx = load_golden("vae_vid5x64")
    _, _, xg = golden_setup(fx)
    _orig = torch.randn
    try:
        torch.randn = lambda *a, **k: fx["noise"].clone() if tuple(a[0]) == tuple(fx["noise"].shape) else _orig(*a, **k)
        z = m.encode_batch([xs[1].to(cuda), xg[0].to(cuda)])[1]
    finally:
        torch.randn = _orig
    check_sub(fx["z"], z[None], 1e-4, "vae latent")
    check_sub(fx["rec"], m.decode_batch([z.permute(1, 2, 3, 0)])[0][None], PIX_TOL, "vae reconstruction")


def test_encode_batch_slot_replay_and_layouts_with_equal_rows(cuda):
    cfg, sd, _ = golden_setup(load_golden("img64"))
    m = build_model(cfg, sd, cuda, "f16x3")
    eng = m.engine()
    xs = [W.synthetic_input((1, 3, 5, 64, 64), 21)[0], W.synthetic_input((1, 3, 64, 64), 22)[0],
          W.synthetic_input((1, 3, 9, 64, 64), 23)[0]]                     # T' = 2, 1, 3: 6 frames
    runs = [m.encode_batch(xs) for _ in range(3)]
    ws = eng._workspace(6 * 64)
    graphs = list(ws.graphs_of("encode_batch").values())
    assert graphs and isinstance(graphs[0], tuple), "the second call of a layout captures a graph, the third replays it"
    for r in runs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(runs[0], r))
    decs = [m.decode_batch(runs[0]) for _ in range(3)]
    for d in decs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(decs[0], d))
    # same row count, other layout (T' = 3, 3): runs on its own and returns its own result
    ys = [W.synthetic_input((1, 3, 9, 64, 64), 24)[0], W.synthetic_input((1, 3, 9, 64, 64), 25)[0]]
    zs = [W.synthetic_input((1, 3, 5, 64, 64), 26)[0], W.synthetic_input((1, 3, 13, 64, 64), 27)[0]]   # T' = 2, 4
    for batch in (ys, zs, ys, zs, ys):
        got = m.encode_batch(batch)
        for x, g in zip(batch, got):
            assert torch.equal(g, m.encode(x[None].to(cuda), False)[0])
        rec = m.decode_batch(got)
        for g, r in zip(got, rec):
            assert torch.equal(r, m.decode(g[None], False)[0])
    assert m.encode_batch([]) == [] and m.decode_batch([]) == [] and m.decode_u8_batch([]) == []


def test_errors_raise_before_launch(cuda):
    from omnitokenizer_b200 import _cabi
    cfg = oo.Config()
    m = build_model(cfg, W.make_state_dict(cfg, 0), cuda, "fp32")
    ok = [torch.zeros(3, 64, 64, device=cuda), torch.zeros(3, 5, 64, 64, device=cuda)]
    n0 = _cabi.launch_count
    usage = m.codebook.codebook_usage.clone()
    with pytest.raises(ValueError, match="same frame size"):
        m.encode_batch(ok + [torch.zeros(3, 128, 128, device=cuda)])
    with pytest.raises(ValueError, match="channels"):
        m.encode_batch(ok + [torch.zeros(4, 5, 64, 64, device=cuda)])
    with pytest.raises(AssertionError, match="divisible by temporal patch size"):
        m.encode_batch(ok + [torch.zeros(3, 6, 64, 64, device=cuda)])
    with pytest.raises(NotImplementedError, match="at most 17 latent frames"):
        m.encode_batch([torch.zeros(3, 69, 64, 64, device=cuda)] + ok)
    with pytest.raises(ValueError, match="token grid"):
        m.encode_batch([torch.zeros(3, 5, 32, 32, device=cuda)])
    with pytest.raises(ValueError, match="square"):
        m.encode_batch([torch.zeros(3, 5, 64, 128, device=cuda)])
    codes = [torch.zeros(8, 8, dtype=torch.int64, device=cuda), torch.zeros(2, 8, 8, dtype=torch.int64, device=cuda)]
    with pytest.raises(NotImplementedError, match="at most 17 latent frames"):
        m.decode_batch(codes + [torch.zeros(18, 8, 8, dtype=torch.int64, device=cuda)])
    with pytest.raises(ValueError, match="same token grid"):
        m.decode_u8_batch(codes + [torch.zeros(2, 16, 16, dtype=torch.int64, device=cuda)])
    assert _cabi.launch_count == n0, "a rejected batch launched kernels"
    assert m.codebook.call_cnt == 0 and torch.equal(m.codebook.codebook_usage, usage)


def test_layout_state_and_decode_batch_slots_stay_bounded(cuda):
    """The same lengths in other orders reuse one layout (no engine-wide table grows); decode_batch and decode_u8_batch
    alternating on one layout each keep their own outputs and reach graph replay."""
    cfg, sd, _ = golden_setup(load_golden("img64"))
    m = build_model(cfg, sd, cuda, "f16x3")
    eng = m.engine()
    base = [W.synthetic_input((1, 3, 5, 64, 64), 31)[0], W.synthetic_input((1, 3, 64, 64), 32)[0],
            W.synthetic_input((1, 3, 9, 64, 64), 33)[0], W.synthetic_input((1, 3, 5, 64, 64), 34)[0]]
    first = m.encode_batch(base)
    n_tables = len(eng._tables)
    for perm in ([3, 2, 1, 0], [1, 0, 3, 2], [2, 3, 0, 1], [0, 2, 1, 3], [3, 1, 2, 0]):
        got = m.encode_batch([base[i] for i in perm])
        for k, i in enumerate(perm):
            assert torch.equal(got[k], first[i])
    assert len(eng._tables) == n_tables
    ws = eng._workspace(8 * 64)
    assert len(ws.layout_tables) == 1
    recs, recs8 = [], []
    for _ in range(3):
        recs.append(m.decode_batch(first))
        recs8.append(m.decode_u8_batch(first))
    for r, r8 in zip(recs[1:], recs8[1:]):
        assert all(torch.equal(a, b) for a, b in zip(recs[0], r)) and all(torch.equal(a, b) for a, b in zip(recs8[0], r8))
    dec = [ws.graphs_of(slot) for slot in ("decode_batch", "decode_batch_u8")]
    assert all(len(g) == 1 and all(isinstance(v, tuple) for v in g.values()) for g in dec), "both output forms replay a graph"
    assert len(ws.layout_tables) == 1


def test_encode_batch_graph_survives_other_encode_inputs(cuda):
    """encode and encode_u8 at other shapes of the same row count replace only their own static inputs: encode_batch
    keeps replaying the graph it captured."""
    cfg, sd, _ = golden_setup(load_golden("img64"))
    m = build_model(cfg, sd, cuda, "f16x3")
    eng = m.engine()
    xs = [W.synthetic_input((1, 3, 5, 64, 64), 41)[0], W.synthetic_input((1, 3, 64, 64), 42)[0],
          W.synthetic_input((1, 3, 9, 64, 64), 43)[0]]                     # T' = 2, 1, 3: 6 frames
    runs = [m.encode_batch(xs) for _ in range(3)]
    ws = eng._workspace(6 * 64)
    (g,) = ws.graphs_of("encode_batch").values()
    assert isinstance(g, tuple)
    m.encode(W.synthetic_input((2, 3, 9, 64, 64), 44).to(cuda), False)      # 2 x T' = 3: 6 frames
    frames = torch.randint(0, 256, (6, 64, 64, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(45))
    m.encode_u8(frames.to(cuda), True)                                      # 6 images
    assert len(eng._ws) == 1 and ws.graphs_of("encode") and ws.graphs_of("encode_u8")
    runs.append(m.encode_batch(xs))
    (g_after,) = ws.graphs_of("encode_batch").values()
    assert g_after is g, "encode_batch captured its graph again"
    assert all(torch.equal(a, b) for a, b in zip(runs[0], runs[-1]))


def test_long_clip_in_a_packed_batch_without_temporal_blocks(cuda):
    """A model without temporal blocks encodes clips past 17 latent frames on their own, but a batch of different lengths
    goes through the layout tables (1..17 frames per sample): rejected before any launch."""
    import omnitokenizer_b200 as ob
    from omnitokenizer_b200 import _cabi
    from tests.util import namespace_from_cfg
    cfg = oo.Config()
    m = ob.OmniTokenizer_VQGAN(namespace_from_cfg(cfg, temporal_depth=0))
    m.load_state_dict(W.make_state_dict(cfg, 0), strict=False)
    m.codebook._need_init = False
    m = m.to(cuda).eval()
    n0 = _cabi.launch_count
    with pytest.raises(NotImplementedError, match="at most 17 latent frames"):
        m.encode_batch([torch.zeros(3, 64, 64, device=cuda), torch.zeros(3, 69, 64, 64, device=cuda)])
    with pytest.raises(NotImplementedError, match="at most 17 latent frames"):
        m.decode_batch([torch.zeros(8, 8, dtype=torch.int64, device=cuda), torch.zeros(18, 8, 8, dtype=torch.int64, device=cuda)])
    assert _cabi.launch_count == n0 and m.codebook.call_cnt == 0
