"""The f16x1 throughput mode on the GPU: the single-product GEMM (omt_linear_h1) and spatial attention core
(omt_attn_spatial_h1) across their walks, the model against the golden vectors within the bounds the CPU numerics model
(tests/f16x1_model.py) predicts, the exact invariants the mode keeps (batch independence, batched and uint8 entry
points, graph replay, determinism), isolation from the other modes in one process, and argument checks.

GEMM walk: the exact-grid operands of test_gpu_gemm_walk.py with their lo planes left out.  Every hi.hi product and
partial sum is exact in fp32, so the kernel's one possible result is fp64's, bit for bit, in every epilogue that writes
fp32.  Epilogues that write fp16 planes round once more, to 2^-11 of the value.
"""
import types

import pytest
import torch

from omnitokenizer_b200 import layout as L
from oracle import omni_oracle as oo
from oracle import weights as W
from oracle.u8_norm import video_norm
from tests import test_gpu_attn_walk as aw
from tests import test_gpu_gemm_walk as gw
from tests.f16x1_model import mm_f16x1, provable_near_tie
from tests.util import build_model, check_sub, golden_setup, load_golden

pytestmark = pytest.mark.gpu
LO_FIELDS = ("a_lo", "a2_lo", "w_lo", "u_lo")


def _cabi():
    return gw._cabi()


def _h1_cabi():
    """The binding with linear_h routed to omt_linear_h1 and the lo planes left out: the existing walk cases launch it."""
    cabi = _cabi()

    def linear_h(**kw):
        cabi.linear_h("omt_linear_h1", **{k: v for k, v in kw.items() if k not in LO_FIELDS})

    return types.SimpleNamespace(linear_h=linear_h, call=cabi.call, EPI_NONE=cabi.EPI_NONE, EPI_GEGLU=cabi.EPI_GEGLU,
                                 EPI_QKV=cabi.EPI_QKV, EPI_QKV_PLANES=cabi.EPI_QKV_PLANES)


@pytest.fixture
def hi_only(monkeypatch):
    """Exact-grid operands with zero lo planes: the fp64 reference of test_gpu_gemm_walk.py is then hi . hi."""
    orig = gw.grid_operand

    def grid(rows, cols, seed, dev, form, amp=2):
        t = orig(rows, cols, seed, dev, form, amp)
        return (t[0], torch.zeros_like(t[1])) if form in ("rs", "uniform", "nacc2") else t

    monkeypatch.setattr(gw, "grid_operand", grid)


def _h1_geglu(dev, form, T, K, n_list, tail, static):
    M, N = gw._shape(T, n_list, tail)
    ku = N // 2
    inner = 1365 if ku == 1408 else ku - 11
    amp = 1 if form == "nacc2" else 2
    a = gw.grid_operand(M, K, 21, dev, form, amp)[0]
    w = L.pack_geglu(gw.grid_operand(2 * inner, K, 22, dev, form, amp)[0], inner, ku)
    ars = gw._scales(form, "geglu", M, 23, dev)
    y = a.double() @ w.double().t()
    kw = dict(a_hi=a, lda=K, w_hi=L.pad_rows(w, 256))
    if form == "rs":
        y = y * (ars.double() * gw.W_SCALE)[:, None]
        kw.update(a_rs=ars, w_scale=gw.W_SCALE)
    assert torch.equal(y.float().double(), y)
    val, gate = y[:, 0::2], y[:, 1::2]
    want = gw.gelu64(gate) * val
    us = L.pow2_scale(float(want.abs().max()) * 4.0) if static else 0.0
    ldu = ku + 24
    ub = gw._f16_buf(PRE + M + POST, ldu, dev)
    cabi = _cabi()
    gw._launch3(lambda: cabi.linear_h("omt_linear_h1", u_hi=ub[0, PRE:], ldu=ldu, M=M, N=N, K=K,
                                      epilogue=cabi.EPI_GEGLU, u_scale=us, **kw), [ub], lambda: ub.fill_(gw.SENT16))
    hi = ub[0, PRE: PRE + M, :ku].view(torch.float16).double()
    assert not hi.isnan().any(), "NaN left inside the U plane"
    got = hi / us if static else hi
    # fp32 GEGLU (test_gpu_gemm_walk.py's 2^-20 bound), then one rounding to fp16: 2^-11 of the value above the
    # subnormal floor 2^-25 (of the scaled value)
    tol = 2.0 ** -20 * val.abs() * gate.abs() + 2.0 ** -11 * want.abs() + 2.0 ** -25 / (us if static else 1.0)
    err = (got[:, :inner] - want[:, :inner]).abs() - tol[:, :inner]
    assert (err <= 0).all(), f"GEGLU hi plane off by more than its bound: {(got - want).abs().max().item():.3e}"
    assert torch.count_nonzero(ub[0, PRE: PRE + M, inner:ku]).item() == 0, "padding columns are not exact zeros"
    mask = torch.zeros(ub.shape, dtype=torch.bool, device=dev)
    mask[0, PRE: PRE + M, :ku] = True                 # the lo plane buffer is never written
    gw._check_guard(ub, mask, gw.SENT16, "U planes")
    return M, N


def _h1_planes(dev, T, K, n_list, tail, tokens):
    M, N = gw._shape(T, n_list, tail)
    qk, n_split = gw._qkv_layout(N)
    a = gw.grid_operand(M, K, 31, dev, "rs")[0]
    ars = gw._scales("rs", "qkv", M, 32, dev)
    w = gw.grid_operand(N, K, 35, dev, "rs")[0]
    kw = dict(a_hi=a, a_rs=ars, w_scale=gw.W_SCALE, lda=K, w_hi=L.pad_rows(w, 256))
    z = (a.double() @ w.double().t()) * (ars.double() * gw.W_SCALE)[:, None]
    if n_split:
        a2 = gw.grid_operand(M, K, 33, dev, "rs")[0]
        a2rs = gw._scales("rs", "qkv", M, 34, dev)
        kw.update(a2_hi=a2, a2_rs=a2rs, n_split=n_split)
        z[:, n_split:] = ((a2.double() @ w.double().t()) * (a2rs.double() * gw.W_SCALE)[:, None])[:, n_split:]
    assert torch.equal(z.float().double(), z)
    g = gw._gen(36, dev)
    qs, ks = 0.5 + torch.rand(64, generator=g, device=dev), 0.5 + torch.rand(64, generator=g, device=dev)
    cos, sin = [t.to(dev) for t in L.rope_tables(tokens, 64)]
    qk_want, sc = gw._qk_ref(z, qk, qs, ks, cos, sin, tokens)
    hv = (N - qk) // 64
    qps, kps = L.pow2_scale(float(qs.max())), L.pow2_scale(float(ks.max()))
    ldu = N + 40
    pb = gw._f16_buf(PRE + M + POST, ldu, dev)
    vinv = torch.empty(hv * M + 7, device=dev)

    def reset():
        pb.fill_(gw.SENT16)
        vinv.view(torch.int32).fill_(gw.SENT32)

    cabi = _cabi()
    gw._launch3(lambda: cabi.linear_h("omt_linear_h1", u_hi=pb[0, PRE:], ldu=ldu, M=M, N=N, K=K,
                                      epilogue=cabi.EPI_QKV_PLANES, q_scale=qs, k_scale=ks, rope_cos=cos, rope_sin=sin,
                                      qk_cols=qk, tokens=tokens, q_plane_scale=qps, k_plane_scale=kps, vinv=vinv, **kw),
                [pb, vinv], reset)
    hi = pb[0, PRE: PRE + M, :N]
    assert not hi.view(torch.float16).isnan().any()
    ps = torch.tensor([qps] * (qk // 2) + [kps] * (qk // 2), device=dev, dtype=torch.float64)
    val = hi[:, :qk].view(torch.float16).double() / ps
    tol = 2.0 ** -18 * sc
    err = (val - qk_want).abs()
    assert (err <= tol + 2.0 ** -11 * (qk_want.abs() + tol) + 2.0 ** -25 / ps).all(), "q / k hi planes off"
    vh, _, vi = L.split_rows_rs(z[:, qk:].float().reshape(M * hv, 64))
    assert torch.equal(hi[:, qk:], vh.view(torch.int16).reshape(M, N - qk)), "v hi plane differs from the host twin"
    assert torch.equal(vinv[: hv * M].view(hv, M), vi.view(M, hv).t()), "vinv differs from the host twin"
    mask = torch.zeros(pb.shape, dtype=torch.bool, device=dev)
    mask[0, PRE: PRE + M, :N] = True
    gw._check_guard(pb, mask, gw.SENT16, "q | k | v planes")
    vmask = torch.zeros(vinv.shape, dtype=torch.bool, device=dev)
    vmask[: hv * M] = True
    gw._check_guard(vinv, vmask, gw.SENT32, "vinv")
    return M, N


PRE, POST = gw.PRE, gw.POST

# (form, epilogue, T, K, candidate N, rows in the last m block, options): every GEMM the f16x1 engine launches --
# patch embed (rs, bias, row maps), window qkv / to_pixels (rs), out-proj / window proj / FF2 (2^11 form "nacc2" or
# "uniform", bias, residual), FF1 (GEGLU in both U forms), the dual-A QKV GEMM (planes, and fp32 for the fallback)
SWEEP = [
    ("rs", "plain", "1", 64, [64], 1, dict(bias=True, res="sep")),
    ("rs", "plain", "S-1", 128, [96], 64, dict(bias=True, res="sep", amap=True)),
    ("rs", "plain", "S", 192, [512], 96, dict(bias=True, res="inplace", cmap=True)),
    ("rs", "plain", "S+1", 256, [896, 128], 1, dict(dual=True)),
    ("rs", "plain", "2S+1", 256, [192, 768, 128], 64, dict(bias=True, amap=True, cmap=True)),
    ("uniform", "plain", "3S+1", 1408, [544, 640, 128], 64, dict(res="inplace")),
    ("nacc2", "plain", "S+1", 512, [512, 128], 127, dict(bias=True, res="inplace")),
    ("nacc2", "plain", "2S+1", 64, [64], 64, dict(res="sep")),
    ("rs", "geglu", "2S+1", 256, [2816, 128], 64, {}),
    ("rs", "geglu_us", "S", 192, [896, 128], 127, {}),
    ("nacc2", "geglu", "S-1", 128, [2816, 128], 128, {}),
    ("nacc2", "geglu", "3S+1", 64, [128], 1, {}),
    ("rs", "qkv", "1", 128, [1536, 640, 128], 64, dict(tokens=96)),
    ("rs", "qkv", "2S+1", 64, [640, 1536, 128], 1, dict(tokens=96)),
    ("rs", "planes", "S", 192, [1536, 896, 640], 64, dict(tokens=96)),
    ("rs", "planes", "S+1", 192, [896, 1536, 640], 127, dict(tokens=96)),
    ("rs", "planes", "2S+1", 512, [1536, 896, 640], 128, dict(tokens=128)),
]


@pytest.mark.parametrize("form,epi,t,K,n_list,tail,opt", SWEEP,
                         ids=[f"{c[0]}-{c[1]}-T{c[2]}-K{c[3]}" + ("-" + "-".join(sorted(c[6])) if c[6] else "")
                              for c in SWEEP])
def test_gemm_tile_walk(cuda, hi_only, form, epi, t, K, n_list, tail, opt):
    T = gw.T_KEYS[t](gw._sms())
    if epi == "plain":
        M, N = gw._case_plain(_h1_cabi(), cuda, form, T, K, n_list, tail, opt)
    elif epi == "qkv":
        M, N = gw._case_qkv(_h1_cabi(), cuda, T, K, n_list, tail, opt, rope=True, planes=False)
    elif epi == "planes":
        M, N = _h1_planes(cuda, T, K, n_list, tail, opt["tokens"])
    else:
        M, N = _h1_geglu(cuda, form, T, K, n_list, tail, epi == "geglu_us")
    assert ((M + 127) // 128) * ((N + 127) // 128) == T


# ---- spatial attention core -----------------------------------------------------------------------------------------

class H1Problem(aw.Problem):
    """test_gpu_attn_walk.Problem launched on the hi planes alone; the reference takes the values the hi planes hold."""

    def run(self, o=None, o_hi=None, o_lo=None, ldo=None, s0=0, s1=None):
        assert o_lo is None
        s1 = self.nseq if s1 is None else s1
        r0, r1 = s0 * self.N, s1 * self.N
        ld = self.H * 64
        qh, kh, vh = (self.planes[i][r0:r1] for i in (0, 2, 4))
        vinv = self.vinv[:, r0:r1].contiguous()
        _cabi().call("omt_attn_spatial_h1", qh, ld, kh, ld, vh, ld, vinv, self.qs * self.ks, o, o_hi, ldo, s1 - s0,
                     self.N, self.H, 8.0)

    def reference(self, dev):
        """(fp64 softmax(8 q k^T) v, fp64 softmax(8 q k^T) |v|) on the hi-plane values."""
        M, H = self.M, self.H
        f16 = lambda t: t.view(torch.float16).double().cpu()
        q = (f16(self.planes[0]) / self.qs).view(M, H, 64)
        k = (f16(self.planes[2]) / self.ks).view(M, H, 64)
        v = (f16(self.planes[4]).view(M, H, 64) * self.vinv.cpu().double().t()[:, :, None])
        shp = (self.nseq, self.N, H, 64)
        qq, kk, vv = (t.reshape(shp).permute(0, 2, 1, 3).to(dev) for t in (q, k, v))
        out = torch.empty(self.nseq, H, self.N, 64, dtype=torch.float64, device=dev)
        mag = torch.empty_like(out)
        for s in range(self.nseq):
            p = torch.softmax((qq[s] @ kk[s].transpose(-1, -2)) * 8.0, dim=-1)
            out[s], mag[s] = p @ vv[s], p @ vv[s].abs()
        return [t.permute(0, 2, 1, 3).reshape(M, H * 64) for t in (out, mag)]


def _attn_walk(p, dev, what):
    cols = p.H * 64
    ldo = cols + 8
    runs = []
    for _ in range(3):
        buf = aw._f32_buf(p.M, ldo, dev)
        p.run(o=buf[PRE:], ldo=ldo)
        torch.cuda.synchronize()
        aw._check_guards(buf, p.M, cols, aw.SENT32)
        runs.append(buf)
    for b in runs[1:]:
        assert torch.equal(b.view(torch.int32), runs[0].view(torch.int32)), f"{what}: launches differ"
    o = runs[0][PRE:PRE + p.M, :cols]
    assert not bool(torch.isnan(o).any()), f"{what}: NaN left inside the output"
    want, mag = p.reference(dev)
    # test_gpu_attn_walk.py's fp32-accumulation bound, plus P'' rounded to fp16: 2^-11 of each p_j |v_j|
    rel = 2e-5 if p.N <= 1024 else 6e-5
    tol = rel * want.abs().amax(dim=1, keepdim=True).clamp_min(1e-3) + 2.0 ** -11 * 1.01 * mag
    excess = ((o.double() - want).abs() - tol).max().item()
    assert excess <= 0, f"{what}: error exceeds its bound by {excess:.3e}"
    # O as a hi plane: fp16(o); the lo buffer stays untouched
    op = aw._f16_buf(p.M, ldo, dev)
    p.run(o_hi=op[0, PRE:], ldo=ldo)
    torch.cuda.synchronize()
    aw._check_guards(op[:1], p.M, cols, aw.SENT16)
    assert bool((op[1] == aw.SENT16).all()), f"{what}: the lo plane buffer was written"
    hi = op[0, PRE:PRE + p.M, :cols].view(torch.float16)
    assert torch.equal(hi, o.half()), f"{what}: O hi plane is not fp16 of the fp32 output"


@pytest.mark.parametrize("T", list(aw.T_KEYS))
def test_attn_item_counts_n128(cuda, T):
    items = aw.T_KEYS[T](gw._sms())
    H = next(h for h in (8, 4, 2, 1) if items % h == 0)
    _attn_walk(H1Problem(items // H, 128, H, 300 + items, cuda), cuda, f"N=128 items={items} heads={H}")


@pytest.mark.parametrize("ramp", [False, True])
def test_attn_long_sequences_n4096(cuda, ramp):
    _attn_walk(H1Problem(2, 4096, 8, 77, cuda, ramp=ramp), cuda, f"N=4096 ramp={ramp}")


def test_attn_placement_invariance(cuda):
    N, H = 256, 8
    per_seq = H * N // 128
    nseq = (2 * gw._sms() + 1 + per_seq - 1) // per_seq + 1
    p = H1Problem(nseq, N, H, 91, cuda, ramp=True)
    cols = p.H * 64
    whole = torch.empty(p.M, cols, device=cuda)
    p.run(o=whole, ldo=cols)
    parts = torch.empty(p.M, cols, device=cuda)
    for s0, s1 in ((0, 1), (1, 4), (4, nseq - 1), (nseq - 1, nseq)):
        p.run(o=parts[s0 * N:], ldo=cols, s0=s0, s1=s1)
    torch.cuda.synchronize()
    assert torch.equal(whole.view(torch.int32), parts.view(torch.int32))


# ---- the model against the goldens ----------------------------------------------------------------------------------

def _f16x1_model(cfg, sd, cuda, monkeypatch):
    monkeypatch.setenv("OMT_MATH", "f16x1")
    m = build_model(cfg, sd, cuda)
    assert m.engine().h1
    return m


def _video(x):
    return x.unsqueeze(2) if x.ndim == 4 else x


@pytest.mark.parametrize("name", ["img64", "vid5x64", "vid9x128_b2", "img256_cfg1", "cnn_vid5x64"])
def test_vq_goldens_within_model_bounds(cuda, name, monkeypatch):
    fx = load_golden(name)
    cfg, sd, x = golden_setup(fx)
    is_image = x.ndim == 4
    m = _f16x1_model(cfg, sd, cuda, monkeypatch)
    eng = m.engine()
    ws, _ = eng.encode(_video(x).to(cuda), "vq")
    idx = ws.idx[: ws.M].cpu()
    z_gpu = eng.z_view(ws).cpu().clone()
    ref = fx["idx"].long().reshape(-1)
    flipped = (idx != ref).nonzero().flatten()
    with torch.no_grad():
        h, _ = oo.encoder(sd, cfg, x)
        z = h.reshape(-1, h.shape[-1])
        if cfg.l2_code:
            z = z / z.norm(dim=1, keepdim=True).clamp_min(1e-12)
    assert len(flipped) <= 0.01 * ref.numel(), f"{len(flipped)}/{ref.numel()} codes differ"
    if len(flipped):
        ok = provable_near_tie(z[flipped], z_gpu[flipped], sd["codebook.embeddings"], ref[flipped], idx[flipped])
        assert ok.all(), f"flipped codes that are not near-ties: {flipped[~ok].tolist()}"
    rec = m.decode(fx["idx"].long().to(cuda), is_image)
    err = check_sub(fx["rec"], rec, 5e-3, "reconstruction")
    monkeypatch.setattr(oo, "MATMUL_MODEL", mm_f16x1)
    with torch.no_grad():
        model_err = check_sub(fx["rec"], oo.decode(sd, cfg, fx["idx"].long(), is_image), 1.0, "model")
    print(f"{name} [f16x1]: flips {len(flipped)}/{ref.numel()}, max |dpx| {err:.2e} (model {model_err:.2e})")
    assert err <= 3 * model_err, f"max |dpx| {err:.2e} > 3 x the model's {model_err:.2e}"


@pytest.mark.parametrize("name", ["vae_vid5x64", "vae_img64"])
def test_vae_moments_within_model_bounds(cuda, name, monkeypatch):
    """VAE: the moments (mean, logvar) before the noise, against 3x the model's error."""
    fx = load_golden(name)
    cfg, sd, x = golden_setup(fx)
    m = _f16x1_model(cfg, sd, cuda, monkeypatch)
    eng = m.engine()
    ws, _ = eng.encode(_video(x).to(cuda), "raw")
    got = eng.z_view(ws).cpu().clone()
    with torch.no_grad():
        h = oo.encoder(sd, cfg, x)[0]
        monkeypatch.setattr(oo, "MATMUL_MODEL", mm_f16x1)
        hm = oo.encoder(sd, cfg, x)[0]
    h, hm = h.reshape(got.shape), hm.reshape(got.shape)
    err, model_err = (got - h).abs().max().item(), (hm - h).abs().max().item()
    print(f"{name} [f16x1]: moments max |d| {err:.2e} (model {model_err:.2e})")
    assert err <= 3 * model_err


# ---- exact invariants in f16x1 --------------------------------------------------------------------------------------

def _cfg_model(cuda, monkeypatch, seed=2):
    cfg = oo.Config()
    return _f16x1_model(cfg, W.make_state_dict(cfg, seed), cuda, monkeypatch)


def test_batch_independence_and_determinism(cuda, monkeypatch):
    """128 x 128 frames (256 tokens: the single-product attention core runs) and 64 x 64 ones (64 tokens: the fp32
    fallback core): a B = 3 batch equals each sample alone, and two runs agree, bit for bit."""
    m = _cfg_model(cuda, monkeypatch)
    for side in (128, 64):
        x = W.synthetic_input((3, 3, 5, side, side), 9).to(cuda)
        full = m.encode(x, False)
        assert torch.equal(full, m.encode(x, False))
        rf = m.decode(full, False)
        assert torch.equal(rf, m.decode(full, False))
        for i in range(3):
            part = m.encode(x[i:i + 1], False)
            assert torch.equal(part, full[i:i + 1]), f"{side}px sample {i}: codes differ from the batch"
            assert torch.equal(m.decode(part, False), rf[i:i + 1]), f"{side}px sample {i}: pixels differ"


def test_batched_entry_points_equal_solo(cuda, monkeypatch):
    m = _cfg_model(cuda, monkeypatch)
    xs = [W.synthetic_input((1, 3, t, 128, 128), 20 + t)[0].to(cuda) for t in (5, 1, 9)]
    xs[1] = xs[1][:, 0]                                 # an image
    codes = m.encode_batch(xs)
    solo = [m.encode(x[None], x.ndim == 3)[0] for x in xs]
    solo = [s[0] if x.ndim == 3 else s for s, x in zip(solo, xs)]     # an image's codes come as (1, h, w)
    for c, s in zip(codes, solo):
        assert torch.equal(c, s)
    recs, u8 = m.decode_batch(codes), m.decode_u8_batch(codes)
    for c, r, r8, x in zip(codes, recs, u8, xs):
        img = x.ndim == 3
        e = c.reshape(1, 1, *c.shape) if img else c[None]
        assert torch.equal(r, m.decode(e, img)[0])
        assert torch.equal(r8, m.decode_u8(e, img)[0])


def test_encode_u8_equals_encode(cuda, monkeypatch):
    m = _cfg_model(cuda, monkeypatch)
    frames = torch.randint(0, 256, (2, 5, 128, 128, 3), generator=torch.Generator().manual_seed(4), dtype=torch.uint8)
    assert torch.equal(m.encode_u8(frames.to(cuda), False), m.encode(video_norm(frames).to(cuda), False))


def test_graph_replay_equals_eager(cuda, monkeypatch):
    """The first call of a shape runs eagerly, the second captures a graph, the third replays it."""
    m = _cfg_model(cuda, monkeypatch)
    x = W.synthetic_input((2, 3, 5, 128, 128), 31).to(cuda)
    codes = [m.encode(x, False) for _ in range(3)]
    recs = [m.decode(codes[0], False) for _ in range(3)]
    for c in codes[1:]:
        assert torch.equal(c, codes[0])
    for r in recs[1:]:
        assert torch.equal(r, recs[0])


def test_modes_do_not_leak(cuda, monkeypatch):
    """An f16x3 model, then an f16x1 engine in the same process, then the f16x3 model again: identical bits."""
    cfg = oo.Config()
    sd = W.make_state_dict(cfg, 3)
    x = W.synthetic_input((2, 3, 5, 128, 128), 41).to(cuda)
    monkeypatch.setenv("OMT_MATH", "f16x3")
    m3 = build_model(cfg, sd, cuda)
    c0 = m3.encode(x, False)
    r0 = m3.decode(c0, False)
    m1 = _f16x1_model(cfg, sd, cuda, monkeypatch)
    c1 = m1.encode(x, False)
    m1.decode(c1, False)
    c2 = m3.encode(x, False)
    r2 = m3.decode(c0, False)
    assert torch.equal(c0, c2) and torch.equal(r0, r2)
    # a fresh f16x3 model built after the f16x1 one agrees too
    monkeypatch.setenv("OMT_MATH", "f16x3")
    m3b = build_model(cfg, sd, cuda)
    assert torch.equal(m3b.encode(x, False), c0) and torch.equal(m3b.decode(c0, False), r0)


# ---- argument checks ------------------------------------------------------------------------------------------------

def _gemm_base(dev):
    M, N, K = 128, 128, 64
    a = torch.zeros(M + 8, K, dtype=torch.int16, device=dev)
    w = torch.zeros(256, K, dtype=torch.int16, device=dev)
    c = torch.full((M, N), float("nan"), device=dev)
    kw = dict(a_hi=a, a_rs=torch.ones(M, device=dev), w_scale=1.0, lda=K, w_hi=w, c=c, ldc=N, M=M, N=N, K=K)
    return kw, c


def test_linear_h1_rejects_bad_arguments(cuda):
    cabi = _cabi()
    kw, c = _gemm_base(cuda)
    a, w = kw["a_hi"], kw["w_hi"]
    u = torch.zeros(2, 128, 64, dtype=torch.int16, device=cuda)
    bad = [
        (dict(a_lo=a), "lo planes must be NULL"),
        (dict(w_lo=w), "lo planes must be NULL"),
        (dict(a2_hi=a, a2_lo=a, a2_rs=kw["a_rs"], n_split=256), "lo planes must be NULL"),
        (dict(epilogue=cabi.EPI_GEGLU, c=None, u_hi=u[0], u_lo=u[1], ldu=64), "lo planes must be NULL"),
        (dict(a_hi=None), "null operand plane"),
        (dict(w_hi=None), "null operand plane"),
        (dict(a_hi=a.view(-1)[1:]), "16-byte aligned"),
        (dict(c=c.view(-1)[1:]), "16-byte aligned"),
        (dict(lda=68), "lda % 8 == 0"),
        (dict(ldc=130), "ldc % 4 == 0"),
        (dict(K=96), "multiple of 64"),
        (dict(epilogue=cabi.EPI_GEGLU, c=None, u_hi=u[0], ldu=60), "ldu % 8 == 0"),
        (dict(w_scale=0.0), "weight scale"),
    ]
    for over, why in bad:
        c.fill_(float("nan"))
        args = dict(kw, **over)
        with pytest.raises(RuntimeError) as e:
            cabi.linear_h("omt_linear_h1", **args)
        assert "omt_linear_h1" in str(e.value) and why in str(e.value), str(e.value)
        torch.cuda.synchronize()
        assert bool(c.isnan().all()), f"{over}: the rejected call wrote C"
    # the three-product entry point still demands its lo planes
    with pytest.raises(RuntimeError, match="omt_linear_h: null operand plane"):
        cabi.linear_h(**kw)
    cabi.linear_h("omt_linear_h1", **kw)                  # and the base block is valid
    torch.cuda.synchronize()
    assert not bool(c.isnan().any())


def test_attn_spatial_h1_rejects_bad_arguments(cuda):
    cabi = _cabi()
    M, H = 256, 2
    q = torch.zeros(M + 8, H * 64, dtype=torch.int16, device=cuda)
    vinv = torch.ones(H, M, device=cuda)
    o = torch.full((M, H * 64), float("nan"), device=cuda)

    def args(**over):
        d = dict(q=q, ldq=128, k=q, ldk=128, v=q, ldv=128, vinv=vinv, ps=1.0, o=o, o_hi=None, ldo=128, n_seq=1, N=256,
                 heads=H)
        d.update(over)
        return (d["q"], d["ldq"], d["k"], d["ldk"], d["v"], d["ldv"], d["vinv"], d["ps"], d["o"], d["o_hi"], d["ldo"],
                d["n_seq"], d["N"], d["heads"], 8.0)

    bad = [(dict(q=None), "null pointer"), (dict(vinv=None), "null pointer"), (dict(o=None), "null pointer"),
           (dict(k=q.view(-1)[1:]), "16-byte aligned"), (dict(o=o.view(-1)[2:]), "16-byte aligned"),
           (dict(ldq=100), "bad leading dims"), (dict(ldo=130), "bad leading dims"),
           (dict(N=192, n_seq=1), "multiple of 128"), (dict(heads=0), "bad arguments"), (dict(ps=0.0), "bad arguments")]
    for over, why in bad:
        o.fill_(float("nan"))
        with pytest.raises(RuntimeError) as e:
            cabi.call("omt_attn_spatial_h1", *args(**over))
        assert "omt_attn_spatial_h1" in str(e.value) and why in str(e.value), str(e.value)
        torch.cuda.synchronize()
        assert bool(o.isnan().all()), f"{over}: the rejected call wrote O"
    cabi.call("omt_attn_spatial_h1", *args())
    torch.cuda.synchronize()
    assert not bool(o.isnan().any())
