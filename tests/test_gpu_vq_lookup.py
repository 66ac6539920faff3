"""The codebook lookup (csrc/vq.cu vq_fused_kernel, through omt_vq_search and omt_vq_fused) checked bit for bit.

Its first-minimum rule has three stages a subtly wrong kernel could get wrong unnoticed: the per-group minimum of each
thread (strict < between groups of 8 codes), the re-evaluation of the winning group (the first code whose distance
equals the group minimum bit for bit), and the merge of the 8 slices of a cluster in ascending order.  The operands sit
on the grids of tests/vq_cases.py, where every distance is exact in fp32 in any order, so the fp64 first argmin is the
only correct index.  Planted tuples put exact ties and 1-ulp near ties inside a group, between groups, at the ends of a
slice, across slice boundaries and across the whole table, on rows at every rows-per-thread slot and owner CTA of a
cluster block, in both launch forms (256-row blocks below the switch at M2 rows, 512-row blocks above it).
Outputs sit in sentinel-filled buffers with guards on both sides; three launches must give the same bits.
"""
import functools

import pytest
import torch

from oracle import omni_oracle as oo
from oracle import weights as W
from tests import vq_cases as V
from tests.util import load_golden, namespace_from_cfg

pytestmark = pytest.mark.gpu

SENT_IDX = -0x5EED
SENT32 = 0x7FBADBAD
SENT_CNT = -0x5EED
PRE, POST = 3, 515          # guard elements before / after each output (POST covers the rest of the last cluster block)
N_CODES = [64, 128, 1024, 2048, 3648, 8192, 16384, 40960]
C = 512


def _cabi():
    from omnitokenizer_b200 import _cabi
    _cabi.load()
    return _cabi


@functools.lru_cache(None)
def _m2():
    """The largest M that takes 2 rows per thread (256-row cluster blocks): the 4-row form would not fill the GPU."""
    return 512 * ((_cabi().device_info()[0] - 1) // 8)


def _ms():
    m2 = _m2()
    return [1, 255, 256, 257, 511, m2, m2 + 1, m2 + 255, 40960, 147456]


def _block(M):
    return 256 if M <= _m2() else 512


class Out:
    """idx [M] (int64), z [M, 8] and counts [n] inside sentinel-filled buffers with guards on both sides."""

    def __init__(self, M, n_codes, dev, z=True, counts=True):
        self.M, self.n = M, n_codes
        self.idx_buf = torch.full((PRE + M + POST,), SENT_IDX, dtype=torch.int64, device=dev)
        self.z_buf = torch.empty(PRE + M + POST, 8, device=dev) if z else None
        if z:
            self.z_buf.view(torch.int32).fill_(SENT32)
        self.cnt_buf = None
        if counts:
            self.cnt_buf = torch.full((PRE + n_codes + POST,), SENT_CNT, dtype=torch.int32, device=dev)
            self.cnt_buf[PRE:PRE + n_codes] = 0

    idx = property(lambda s: s.idx_buf[PRE:PRE + s.M])
    z = property(lambda s: None if s.z_buf is None else s.z_buf[PRE:PRE + s.M])
    counts = property(lambda s: None if s.cnt_buf is None else s.cnt_buf[PRE:PRE + s.n])

    def ptrs(self):
        return (None if self.z_buf is None else self.z_buf[PRE:], self.idx_buf[PRE:],
                None if self.cnt_buf is None else self.cnt_buf[PRE:])

    def check_guards(self, what):
        g = lambda t: torch.cat([t[:PRE].reshape(-1), t[-POST:].reshape(-1)])
        assert bool((g(self.idx_buf) == SENT_IDX).all()), f"{what}: idx written outside rows [0, M)"
        if self.z_buf is not None:
            assert bool((g(self.z_buf.view(torch.int32)) == SENT32).all()), f"{what}: z written outside rows [0, M)"
        if self.cnt_buf is not None:
            assert bool((g(self.cnt_buf) == SENT_CNT).all()), f"{what}: counts written outside [0, n_codes)"


def _search(z, E, e2, out):
    zo, idx, cnt = out.ptrs()
    _cabi().call("omt_vq_search", z, E, e2, out.M, out.n, idx, cnt)


def _fused(x, Wt, b, l2, E, e2, out):
    zo, idx, cnt = out.ptrs()
    _cabi().call("omt_vq_fused", x, x.shape[1], Wt, b, x.shape[1], l2, zo, E, e2, out.M, out.n, idx, cnt)


def _explain(got, want, M, what):
    bad = (got != want).nonzero().flatten()
    rows = bad[:6].tolist()
    blk = _block(M)
    return (f"{what}: {bad.numel()} of {M} rows differ; first rows {rows} (offsets in a {blk}-row block "
            f"{[r % blk for r in rows]}) got {got[bad[:6]].tolist()} want {want[bad[:6]].tolist()}")


def _launch3(run, M, n_codes, dev, want, z_want=None, what=""):
    """Three launches into fresh guarded buffers, counts accumulating in one buffer: identical bits, the expected
    indices (and z), counts == 3 x bincount, guards intact."""
    outs = []
    cnt_out = Out(M, n_codes, dev, z=z_want is not None)
    for i in range(3):
        o = Out(M, n_codes, dev, z=z_want is not None, counts=False)
        o.cnt_buf = cnt_out.cnt_buf
        run(o)
        torch.cuda.synchronize()
        o.check_guards(f"{what} launch {i}")
        outs.append(o)
    o = outs[0]
    assert torch.equal(o.idx, want), _explain(o.idx, want, M, what)
    if z_want is not None:
        assert torch.equal(o.z.view(torch.int32), z_want.view(torch.int32)), f"{what}: z differs from the exact projection"
    for p in outs[1:]:
        assert torch.equal(p.idx, o.idx) and (z_want is None or torch.equal(p.z.view(torch.int32), o.z.view(torch.int32))), \
            f"{what}: launches disagree"
    assert torch.equal(cnt_out.counts.long(), 3 * torch.bincount(want, minlength=n_codes)), f"{what}: counts"


@functools.lru_cache(4)
def _case(n_codes, kind, blk, Mmax):
    """(E, e2, z [Mmax, 8], want [Mmax], planted rows, their indices) on the device for one table and launch form."""
    dev = torch.device("cuda:0")
    if kind == "grid":
        z, E = V.tie_grid(Mmax, n_codes, 100 + n_codes + blk, dev)
        rows = want_p = None
    else:
        E, plants = V.ulp_table(n_codes, kind, n_codes)
        E = E.to(dev)
        z, rows, want_p = V.ulp_rows(Mmax, blk, plants, 7 + blk, dev)
    want = V.ref_argmin(z, E)
    if rows is not None:
        assert torch.equal(want[rows], want_p), "planted winners are not the fp64 first minima"
    return E, V.e2_of(E), z, want, rows, want_p


@pytest.mark.parametrize("kind", V.KINDS + ("grid",))
@pytest.mark.parametrize("n_codes", N_CODES)
def test_first_minimum_sweep(cuda, n_codes, kind):
    """omt_vq_search on z, and omt_vq_fused (l2 = 0) on x, Wt, b whose projection is exactly z, at every M of the sweep."""
    ms = _ms()
    for blk in (256, 512):
        m_form = [M for M in ms if _block(M) == blk]
        Mmax = max(m_form)
        E, e2, z, want, rows, want_p = _case(n_codes, kind, blk, Mmax)
        x, Wt, b = V.grid_projection(z, C, 3)
        for M in m_form:
            what = f"n_codes={n_codes} {kind} M={M}"
            _launch3(lambda o: _search(z[:M], E, e2, o), M, n_codes, cuda, want[:M], what="search " + what)
            _launch3(lambda o: _fused(x[:M], Wt, b, 0, E, e2, o), M, n_codes, cuda, want[:M], z_want=z[:M],
                     what="fused " + what)
        if rows is not None:     # the planted cases were reached at every offset of the block in this form
            assert set((rows % blk).tolist()) == {r for r in V.LROWS if r < blk}


def _rand(shape, seed, scale=1.0):
    return (torch.rand(shape, generator=torch.Generator().manual_seed(seed)) - 0.5) * 2 * scale


def _model_like(M, n_codes, seed, dev):
    """Random x, the model's projection scale and a N(0, 1)-like codebook (oracle/weights.py)."""
    x = _rand((M, C), seed).to(dev)
    Wt, b = _rand((8, C), seed + 1, 0.05).to(dev), _rand((8,), seed + 2, 0.1).to(dev)
    E = (torch.rand((n_codes, 8, 12), generator=torch.Generator().manual_seed(seed + 3)).sum(-1) - 6.0).to(dev)
    return x, Wt, b, E


@pytest.mark.parametrize("n_codes", [1024, 8192])
def test_l2_planted_ties(cuda, n_codes):
    """omt_vq_fused with l2 = 1: z is not exact, so ties are planted by copying the kernel's own z rows into the table at
    every tuple; each planted row must get the first code of its tuple, every row the oracle's index on the kernel's z,
    and z the bits of omt_pre_vq."""
    cabi = _cabi()
    for M in (511, _m2() + 255):
        x, Wt, b, E = _model_like(M, n_codes, 20 + M, cuda)
        zp = torch.empty(M, 8, device=cuda)
        cabi.call("omt_pre_vq", x, C, Wt, b, zp, M, C, 8, 1)
        tup = V.tuples(n_codes)
        rows = V.planted_rows(M, _block(M), 1)[0].tolist()     # one row per tuple: the table holds one z per code
        E2 = E.clone()
        plant = {}
        for t, r in zip(tup, rows):
            E2[list(t)] = zp[r]
            plant[r] = t[0]
        assert len(plant) == len(tup)
        zc = zp.cpu()
        want = oo.codebook(E2.cpu(), zc)["idx"].to(cuda)
        for r, k in plant.items():
            assert int(want[r]) == k, f"oracle: row {r} -> {int(want[r])}, planted {k}"
        _launch3(lambda o: _fused(x, Wt, b, 1, E2, V.e2_of(E2), o), M, n_codes, cuda, want, z_want=zp,
                 what=f"l2 n_codes={n_codes} M={M}")


def test_optional_outputs_and_contention(cuda):
    n_codes, M = 2048, _m2() + 1
    E, e2, z, want, _, _ = _case(n_codes, "tie", 512, 147456)
    x, Wt, b = V.grid_projection(z[:M].contiguous(), C, 3)
    for run in (lambda o: _search(z[:M], E, e2, o), lambda o: _fused(x, Wt, b, 0, E, e2, o)):
        o = Out(M, n_codes, cuda, z=False, counts=False)       # z = NULL, counts = NULL
        run(o)
        torch.cuda.synchronize()
        o.check_guards("NULL outputs")
        assert torch.equal(o.idx, want[:M])
    # every row on one code: M atomic increments of the same counter
    Mc = 40960
    zc = torch.zeros(Mc, 8, device=cuda)
    Ec = E.clone()
    Ec[n_codes - 1] = torch.tensor([float(V.A_PLANT)] + [0.0] * 7, device=cuda)
    for M1 in (Mc, _m2()):
        o = Out(M1, n_codes, cuda)
        _search(zc[:M1], Ec, V.e2_of(Ec), o)
        torch.cuda.synchronize()
        o.check_guards("contention")
        assert bool((o.idx == n_codes - 1).all())
        assert int(o.counts[n_codes - 1]) == M1 and int(o.counts.sum()) == M1


def test_placement_invariance(cuda):
    """One 512-row-block launch equals, bit for bit in idx and z, launches of 256-row-block windows of its rows."""
    n_codes = 8192
    m2 = _m2()
    M = m2 + 600
    x, Wt, b, E = _model_like(M, n_codes, 40, cuda)
    e2 = V.e2_of(E)
    big = Out(M, n_codes, cuda)
    _fused(x, Wt, b, 1, E, e2, big)
    for s in (1, 37, 256, 511):
        for lo, hi in ((0, s), (s, s + m2), (s + m2, M)):
            w = Out(hi - lo, n_codes, cuda)
            _fused(x[lo:hi], Wt, b, 1, E, e2, w)
            torch.cuda.synchronize()
            w.check_guards(f"window [{lo}, {hi})")
            assert torch.equal(w.idx, big.idx[lo:hi]), _explain(w.idx, big.idx[lo:hi], hi - lo, f"window [{lo}, {hi})")
            assert torch.equal(w.z.view(torch.int32), big.z[lo:hi].view(torch.int32)), f"z of window [{lo}, {hi})"
    assert torch.equal(big.counts.long(), torch.bincount(big.idx, minlength=n_codes))


def test_oracle_agreement_at_scale(cuda):
    """40 960 random rows through the fused lookup (l2 = 1): the oracle's argmin on the kernel's own z, every row."""
    n_codes, M = 8192, 40960
    x, Wt, b, E = _model_like(M, n_codes, 50, cuda)
    o = Out(M, n_codes, cuda)
    _fused(x, Wt, b, 1, E, V.e2_of(E), o)
    torch.cuda.synchronize()
    o.check_guards("at scale")
    z, got, Ec = o.z.cpu(), o.idx.cpu(), E.cpu()
    want = torch.cat([oo.codebook(Ec, z[i:i + 4096])["idx"] for i in range(0, M, 4096)])
    bad = (got != want).nonzero().flatten()
    msg = []
    for r in bad[:4].tolist():
        zr = z[r:r + 1]
        d32 = ((zr ** 2).sum(1, keepdim=True) - (2 * zr) @ Ec.t() + (Ec.t() ** 2).sum(0, keepdim=True))[0]
        d64 = ((zr.double() - Ec.double()) ** 2).sum(1)
        g, w = int(got[r]), int(want[r])
        msg.append(f"row {r}: kernel {g} (fp32 {d32[g].item():.9e}, fp64 {d64[g].item():.17e}), "
                   f"oracle {w} (fp32 {d32[w].item():.9e}, fp64 {d64[w].item():.17e})")
    assert bad.numel() == 0, f"{bad.numel()} rows differ from the oracle: " + "; ".join(msg)


@pytest.mark.parametrize("Cp", [64, 256, 512])
@pytest.mark.parametrize("M", [1, 31, 32, 33, 1000])
def test_post_vq(cuda, M, Cp):
    """Gather + post_vq projection: exact on grid operands; the straight-through rows are torch's (E[idx] - z) + z."""
    cabi = _cabi()
    n_codes = 1000
    g = torch.Generator().manual_seed(M * 7 + Cp)
    E = torch.randint(-8, 9, (n_codes, 8), generator=g).float() / 8
    Wq = torch.randint(-4, 5, (Cp, 8), generator=g).float() / 4
    bq = torch.randint(-4, 5, (Cp,), generator=g).float() / 2
    idx = torch.randint(0, n_codes, (M,), generator=g)
    idx[0] = n_codes - 1
    if M > 1:
        idx[-1] = 0
    zr = torch.randn(M, 8, generator=g)                        # straight-through source: any fp32 values
    zg = torch.randint(-8, 9, (M, 8), generator=g).float() / 8
    d = lambda t: t.to(cuda)

    def X_buf():
        t = torch.empty(PRE + M + POST, Cp, device=cuda)
        t.view(torch.int32).fill_(SENT32)
        return t

    def check(X, ref, what):
        assert torch.equal(X[PRE:PRE + M].cpu(), ref.float()), what
        assert bool((X[:PRE].view(torch.int32) == SENT32).all() and (X[PRE + M:].view(torch.int32) == SENT32).all()), \
            f"{what}: rows outside [0, M) written"

    # E[idx] . Wq^T + b: every value a multiple of 2^-5 below 2^6, exact in any order
    X = X_buf()
    cabi.call("omt_post_vq", d(idx), d(E), None, None, None, d(Wq), d(bq), X[PRE:], M, Cp, 8)
    check(X, E[idx].double() @ Wq.double().t() + bq.double(), "gather")
    # straight-through rows (E[idx] - z) + z, bit for bit, and their projection
    X, zq = X_buf(), torch.full((M, 8), float("nan"), device=cuda)
    cabi.call("omt_post_vq", d(idx), d(E), None, d(zr), zq, d(Wq), d(bq), X[PRE:], M, Cp, 8)
    st = (E[idx] - zr) + zr
    assert torch.equal(zq.cpu(), st)
    torch.cuda.synchronize()
    # on a grid z the straight-through row is E[idx] exactly, and so is its projection
    X, zq = X_buf(), torch.full((M, 8), float("nan"), device=cuda)
    cabi.call("omt_post_vq", d(idx), d(E), None, d(zg), zq, d(Wq), d(bq), X[PRE:], M, Cp, 8)
    assert torch.equal(zq.cpu(), E[idx])
    check(X, E[idx].double() @ Wq.double().t() + bq.double(), "straight-through on grid")
    # continuous latents (VAE): rows from zc
    X = X_buf()
    cabi.call("omt_post_vq", None, None, d(zg), None, None, d(Wq), d(bq), X[PRE:], M, Cp, 8)
    check(X, zg.double() @ Wq.double().t() + bq.double(), "zc")


def test_bad_codebook_sizes_raise_before_launch(cuda):
    from omnitokenizer_b200.engine import VQ_MAX_CODES
    M = _m2() + 1               # the 512-row-block form, whose slice bound the engine enforces
    x, Wt, b, _ = _model_like(M, 64, 60, cuda)
    z = torch.zeros(M, 8, device=cuda)
    for n_codes in (96, 100, VQ_MAX_CODES + 64, 65536):
        E = torch.zeros(n_codes, 8, device=cuda)
        e2 = V.e2_of(E)
        for run in (lambda o: _search(z, E, e2, o), lambda o: _fused(x, Wt, b, 1, E, e2, o)):
            o = Out(M, n_codes, cuda)
            with pytest.raises(RuntimeError, match=f"n_codes={n_codes}"):
                run(o)
            torch.cuda.synchronize()
            assert bool((o.idx == SENT_IDX).all()) and bool((o.counts == 0).all()), "a rejected launch wrote outputs"
    # the engine's limit is the largest codebook the 512-row-block form takes
    E, plants = V.ulp_table(VQ_MAX_CODES, "first", 9)
    E = E.to(cuda)
    zu, rows, want = V.ulp_rows(M, 512, plants, 10, cuda)
    o = Out(M, VQ_MAX_CODES, cuda)
    _search(zu, E, V.e2_of(E), o)
    torch.cuda.synchronize()
    assert torch.equal(o.idx, V.ref_argmin(zu, E))


# ---------------------------------------------------------------- the model with codebooks of other sizes

@functools.lru_cache(None)
def _oracle_run(name, n_codes):
    fx = load_golden(name)
    cfg = oo.Config(use_vae=False, patch_embed=fx.get("patch_embed", "linear"), resolution=fx.get("resolution", 256),
                    n_codes=n_codes)
    sd = W.make_state_dict(cfg, fx["wseed"])
    x = W.synthetic_input(fx["shape"], fx["xseed"])
    is_image = x.ndim == 4
    with torch.no_grad():
        idx = oo.encode(sd, cfg, x)
        last = idx.clone()
        last.view(-1)[::3] = n_codes - 1
        return cfg, sd, x, idx, oo.decode(sd, cfg, idx, is_image), last, oo.decode(sd, cfg, last, is_image)


@pytest.mark.parametrize("math", ["fp32", "3xtf32", "f16x3"])
@pytest.mark.parametrize("n_codes", [1000, 2048, 16384])
@pytest.mark.parametrize("name", ["img64", "vid5x64"])
def test_model_codebook_sizes(cuda, monkeypatch, name, n_codes, math):
    import omnitokenizer_b200 as ob
    cfg, sd, x, idx_o, rec_o, last, rec_last = _oracle_run(name, n_codes)
    monkeypatch.setenv("OMT_MATH", math)
    m = ob.OmniTokenizer_VQGAN(namespace_from_cfg(cfg, n_codes=n_codes))
    res = m.load_state_dict(sd, strict=False)
    assert not res.missing_keys and not res.unexpected_keys
    m.codebook._need_init = False
    m = m.to(cuda).eval()
    is_image = x.ndim == 4
    idx = m.encode(x.to(cuda), is_image)
    mism = int((idx.cpu() != idx_o).sum())
    assert mism == 0, f"{mism}/{idx.numel()} code indices differ from the oracle"
    usage = m.codebook.codebook_usage
    assert usage.numel() == n_codes
    assert torch.equal(usage.cpu(), torch.bincount(idx_o.reshape(-1), minlength=n_codes).float() / idx_o.numel())
    err = float((m.decode(idx, is_image).cpu() - rec_o).abs().max())
    assert err <= 1e-3, f"pixels differ by {err:.2e}"
    err = float((m.decode(last.to(cuda), is_image).cpu() - rec_last).abs().max())
    assert err <= 1e-3, f"decoding code n_codes - 1: pixels differ by {err:.2e}"


def test_model_codebook_too_large(cuda):
    import omnitokenizer_b200 as ob
    cfg = oo.Config(n_codes=65536, resolution=64)
    m = ob.OmniTokenizer_VQGAN(namespace_from_cfg(cfg, n_codes=65536))
    m.load_state_dict(W.make_state_dict(cfg, 0), strict=False)
    m = m.to(cuda).eval()
    with pytest.raises(NotImplementedError, match="65536"):
        m.prepare()
