"""The cases of the row-wise kernel tests (tests/rowwise_cases.py), checked on the CPU: the host-selection mirrors reach
every instantiation and PEG tile geometry test_gpu_rowwise.py claims to cover, and the float64 references agree with the
oracle's restatements of the same operations (oracle/omni_oracle.py) within fp32 round-off."""
import pytest
import torch

from oracle import omni_oracle as oo
from tests import rowwise_cases as R


# ---------------------------------------------------------------- mirrors and case tables

def test_ln_cases_reach_every_instantiation():
    """The LayerNorm cases record the (NV, PAIR) the mirror of layernorm_impl picks, and together launch all seven
    compiled kernels, the non-PAIR row-scaled path at C = 512 included."""
    seen = set()
    for C, M, ldx, lds, off, inst32, inst_pl in R.LN_CASES:
        assert R.ln_instantiation(C) == inst32, R.ln_case_id((C, M, ldx, lds, off))
        assert R.ln_instantiation(C, lds, 8 if off % 16 else 16) == inst_pl, R.ln_case_id((C, M, ldx, lds, off))
        seen |= {inst32, inst_pl}
        assert ldx >= C and lds >= C and ldx % 4 == 0 and lds % 4 == 0
    assert seen == {(1, False), (2, True), (2, False), (3, False), (4, True), (4, False), (8, False)}
    Cs = {c[0] for c in R.LN_CASES}
    assert Cs == {4, 100, 128, 256, 384, 512, 640, 768, 1020, 1024}
    assert any(c[0] == 512 and c[3] == 516 for c in R.LN_CASES) and any(c[0] == 512 and c[4] == 8 for c in R.LN_CASES)
    assert any(c[1] % 8 for c in R.LN_CASES) and any(c[2] > c[0] for c in R.LN_CASES)


def test_patch_cases_reach_every_nv():
    Ks, nvs = set(), set()
    for Cin, p, pt, first, K, nv in R.PATCH_CASES:
        assert Cin * (1 if first else pt) * p * p == K
        assert R.patch_nv(K) == nv
        Ks.add(K)
        nvs.add(nv)
    assert {48, 192, 256, 384, 768, 1024} <= Ks and any(K < 128 for K in Ks)
    assert nvs == {2, 6, 8}
    assert {c[0] for c in R.PATCH_CASES} == {1, 3, 4}
    assert {c[1] for c in R.PATCH_CASES} == {4, 8, 16}
    assert {c[2] for c in R.PATCH_CASES} == {1, 2, 4}


def test_peg_mirror_reproduces_the_geometry_table():
    """(TT, HB) at T' = 1, 2 and >= 5 and the kernel for each token row w, as peg_volume_launch derives them.  If this
    fails, the host heuristics changed: update the mirror (rowwise_cases.peg_geometry) and the table together."""
    for w, (g1, g2, g5, kernel) in R.PEG_TABLE.items():
        for T, want in ((1, g1), (2, g2), (5, g5), (9, g5), (17, g5)):
            for causal in (0, 1):
                g = R.peg_geometry(T, w, causal)
                assert (g["TT"], g["HB"]) == want, (w, T, causal, g)
                assert g["kernel"] == kernel, (w, T, g)
                assert g["TT"] * g["HB"] * 8 <= 256 and g["smem"] <= 200 * 1024
    g = R.peg_geometry(5, 192, 1)
    assert g["zrow"] == 9 and g["smem4"] == 124800        # the 121 KB v4 tile
    assert R.peg_geometry(5, 64, 1)["smem4"] <= 69 * 1024  # three CTAs per SM
    assert R.peg_geometry(5, 64, 1, peg_kernel=3)["kernel"] == "v3"


def test_peg_cases_cover_every_geometry():
    v4 = set()
    for w, T, C, h in R.peg_cases():
        g = R.peg_geometry(T, w, 1)
        if g["kernel"] == "v4":
            v4.add((g["TT"], g["HB"]))
        assert (w <= 64) or C == 16
        assert w != 256 or T <= 2
        assert h == w or h % g["HB"] != 0 or g["HB"] == 1, "the last row block of a short frame should be partial"
    assert {hb for _, hb in v4} == {1, 2, 3, 4} and {tt for tt, _ in v4} == {1, 2, 3, 4, 5}
    assert any(R.peg_geometry(T, w, 1)["kernel"] == "v3" for w, T, _, _ in R.peg_cases())
    assert {C for _, _, C, _ in R.peg_cases()} == {16, 512}


def test_families():
    x = R.family_rows(600, 512, 1)
    fam = torch.arange(600) % 6
    assert bool((x[fam == 3] == 0).all())
    const = x[fam == 2]
    assert bool((const == const[:, :1]).all())
    d = x[fam == 1].double()
    assert float((d.mean(1).abs() / d.std(1)).max()) > 50
    p2 = x[fam == 4].abs().amax(1)
    assert torch.equal(torch.frexp(p2).mantissa, torch.full_like(p2, 0.5))
    spread = x[fam == 0].abs().amax(1)
    assert float(spread.max() / spread.min()) > 1e4
    tiny = x[fam == 5]
    assert bool(((tiny[:, ::3].abs() / tiny.abs().amax(1, keepdim=True)) < 2.0 ** -29).all())


# ---------------------------------------------------------------- references vs the oracle

def test_ln_ref_matches_oracle():
    x = R.family_rows(120, 96, 2)
    w, b = R.ln_params(96, 3)
    for bias in (b, None):
        want = oo.layer_norm(x.double(), w.double(), None if bias is None else bias.double())
        got, mag = R.ln_ref(x, w, bias)
        assert float(((got - want).abs() / mag).max()) < 1e-12
    # zero and constant rows give beta exactly
    got, _ = R.ln_ref(x, w, b)
    assert torch.equal(got[2::6].float(), b.expand(20, 96)) and torch.equal(got[3::6].float(), b.expand(20, 96))


@pytest.mark.parametrize("case", R.PATCH_CASES, ids=lambda c: f"Cin{c[0]}-p{c[1]}-pt{c[2]}-first{c[3]}")
def test_patch_refs_match_oracle(case):
    Cin, p, pt, first, K, _ = case
    shape = R.patch_video_shape(Cin, p, pt)
    v = torch.randn(shape, generator=torch.Generator().manual_seed(K))
    f, r = oo.patchify(v, p, pt)
    want = (f if first else r).reshape(-1, K)
    got = R.patchify_ref(v, p, pt, first)
    assert torch.equal(got, want)
    # un-patchify: the inverse permutation, equal to the oracle's inverse Rearranges on its own frames
    back = R.unpatchify_ref(got, shape, p, pt, first)
    full = oo.unpatchify(f, r, Cin, p, pt)
    frames = slice(0, 1) if first else slice(1, None)
    assert torch.equal(back[:, :, frames], full[:, :, frames])
    assert bool((back[:, :, slice(1, None) if first else slice(0, 1)] == 0).all())
    # the LN form of the gather is the LayerNorm reference of the gathered rows
    lw, lb = R.ln_params(K, 5)
    got, mag = R.ln_ref(R.patchify_ref(v, p, pt, first), lw, lb)
    want = oo.layer_norm(want.double(), lw.double(), lb.double())
    assert float(((got - want).abs() / mag).max()) < 1e-12


@pytest.mark.parametrize("temporal", [0, 1])
@pytest.mark.parametrize("causal", [0, 1])
@pytest.mark.parametrize("T,h,w", [(1, 3, 5), (2, 4, 4), (5, 3, 7), (6, 2, 9)])
def test_peg_ref_matches_index_map(T, h, w, temporal, causal):
    """The conv3d formulation (library ops) equals the oracle's index-map restatement; both in float64."""
    B, C = 2, 16
    X = R.peg_input(B, T, h * w, C, 7).double()
    wt, bias = R.peg_params(C, 8)
    got, mag = R.peg_ref(X, wt, bias, h, w, bool(temporal), bool(causal))
    want = oo.peg(X, wt.double(), bias.double(), (h, w), bool(temporal), bool(causal)) + X
    assert float(((got - want).abs() / mag).max()) < 1e-13
    assert not oo.USE_LIBRARY_OPS


def test_qk_prep_ref_matches_oracle():
    M, N, heads = 2 * 64, 64, 3
    t = torch.randn(M, heads * 64, generator=torch.Generator().manual_seed(9))
    sc = torch.rand(64, generator=torch.Generator().manual_seed(10)) + 0.5
    cos, sin = oo.rope_table(N, 64)
    pos = torch.arange(M) % N
    got = R.qk_prep_ref(t, sc, cos[pos], sin[pos])
    want = oo.l2norm(oo.apply_rope(t.double().view(2, N, heads, 64), cos.double(), sin.double())) * sc.double()
    assert float((got - want.reshape(M, -1)).abs().max()) < 1e-12
    got = R.qk_prep_ref(t, sc)
    want = oo.l2norm(t.double().view(M, heads, 64)) * sc.double()
    assert float((got - want.reshape(M, -1)).abs().max()) < 1e-12
    z = torch.zeros(3, 64)
    assert torch.equal(R.qk_prep_ref(z, sc), torch.zeros(3, 64, dtype=torch.float64))


def test_vq_refs():
    x = torch.randn(50, 512, generator=torch.Generator().manual_seed(11))
    Wt, b = torch.randn(8, 512) * 0.05, torch.randn(8) * 0.1
    z, mag = R.pre_vq_ref(x, Wt, b, 1)
    want = oo.l2norm((x @ Wt.t() + b).double())
    assert float((z - want).abs().max()) < 1e-5 and bool((mag >= z.abs()).all())
    E, Wq, bq = torch.randn(64, 8), torch.randn(512, 8), torch.randn(512)
    X, _ = R.post_vq_ref(E[:5], Wq, bq)
    assert float((X - (E[:5] @ Wq.t() + bq).double()).abs().max()) < 1e-5
