"""The evaluation reductions' cases, references and bars (tests/quality_cases.py) on the CPU: the builders give the
sizes, values and padding they claim, the references agree with the oracle / scipy / closed forms, each host model of a
kernel passes its check, and every mutant of it fails that check on the GPU test's cases."""
import math

import numpy as np
import pytest
import torch

from oracle import quality_oracle as qo
from tests import quality_cases as Q


@pytest.fixture(scope="module")
def ssim_u8():
    return Q.ssim_cases("u8")


@pytest.fixture(scope="module")
def ssim_f32():
    return Q.ssim_cases("f32")


@pytest.fixture(scope="module")
def heads():
    return Q.head_cases()


@pytest.fixture(scope="module")
def softmaxes():
    return Q.softmax_cases()


@pytest.fixture(scope="module")
def iss():
    return Q.is_cases()


# ------------------------------------------------------------------------------------------------ builders
def test_ssim_sizes_straddle_the_tile(ssim_u8, ssim_f32):
    """The valid crop takes 1, 2, 32, 33, 43, 64 and 65 in both directions at once: one and two partial outputs, a full
    tile and one past it, and one, two and three tiles per axis."""
    for cases in (ssim_u8, ssim_f32):
        crops = {(c.H - 10, c.W - 10) for c in cases}
        sides = {1, 2, 32, 33, 43, 64, 65}
        assert crops == {(h, w) for h in sides for w in sides}
        assert {h % Q.SS_T for h in sides} == {0, 1, 2, 11} and {-(-h // Q.SS_T) for h in sides} == {1, 2, 3}


def test_ssim_pixel_pairs_cover_tile_edges(ssim_u8):
    """Each one-pixel pair differs in exactly one value, and the differences of a case sit at every (row, column) of
    axis_marks: for 75 these are the tile starts 0, 32, 64, the last outputs 31, 63, the halo ends 41, 73 and 42, 74."""
    assert Q.axis_marks(75) == [0, 31, 32, 41, 42, 63, 64, 73, 74]
    for c in ssim_u8:
        idx = [i for i, k in enumerate(c.kinds) if k == "pixel"]
        pos = set()
        for i in idx:
            d = (c.a[i] != c.b[i]).nonzero()
            assert d.shape[0] == 1 and int(c.sel_a[i]) == int(c.sel_b[i])
            pos.add((int(d[0, 0]), int(d[0, 1])))
        assert pos == {(r, q) for r in Q.axis_marks(c.H) for q in Q.axis_marks(c.W)}, c.name


def test_ssim_tables_and_selections(ssim_u8):
    t = Q.byte_tables()
    assert torch.equal(t[0], torch.arange(256, dtype=torch.float32) / 255)
    assert float((t[1] - t[0]).abs().max()) > 0.1
    for c in ssim_u8:
        combos = {(int(a), int(b)) for a, b, k in zip(c.sel_a, c.sel_b, c.kinds) if k == "noise"}
        assert combos == {(0, 0), (0, 1), (1, 0), (1, 1)}
        for a, b, k in zip(c.sel_a, c.sel_b, c.kinds):
            assert k != "same" or a == b


def test_f32_pairs_leave_the_unit_range(ssim_f32):
    for c in ssim_f32:
        assert float(c.a.min()) < -1 and float(c.a.max()) > 1.5, c.name


def test_head_cases(heads):
    """The NaN padding is in place; every size of the sweep is there; zero vectors and equal pairs are where claimed."""
    seen = set()
    for c in heads:
        assert bool(torch.isnan(c.x[..., c.C:]).all()) and not bool(torch.isnan(c.x[..., :c.C]).any())
        assert (c.Cs - c.C) % 4 == 0
        assert not bool(c.x[0, 0, 0, :c.C].any())
        assert bool(c.x[2 * c.P - 1, -1, -1, :c.C].any()) == (c.P == 1 and c.hw == 1)
        assert bool(c.equal.any()) == (c.P > 3)
        seen.add((c.C, c.Cs > c.C, c.hw, c.P, c.tap))
    assert {s[2] for s in seen} == {1, 15, 16, 17, 37 * 29}
    assert {s[0] for s in seen} == set(Q.HEAD_C) and {s[4] for s in seen} == set(range(5))
    assert all((C, pad, hw, P) in {s[:4] for s in seen} for C in Q.HEAD_C for pad in (False, True)
               for hw in (1, 15, 16, 17, 1073) for P in Q.HEAD_P)


def test_softmax_padding_and_families(softmaxes):
    for c in softmaxes:
        assert bool(torch.isnan(c.xbuf[:, c.N:]).all()) and not bool(torch.isnan(c.x).any())
        if c.rows > 1:
            assert set(c.family.tolist()) == set(range(6))
    assert {(c.N, c.ldx - c.N, c.ldy - c.N, c.rows) for c in softmaxes} == {
        (N, px, py, r) for N in Q.SM_N for px, py in Q.SM_PADS for r in Q.SM_ROWS}


def test_softmax_spread_rows_reach_subnormals_and_zeros(softmaxes):
    """In every spread row of 31 columns or more the fp32 softmax holds subnormal probabilities and probabilities that
    round to 0 although their fp64 value is positive; from 1000 columns on, each row holds at least three of each."""
    for c in softmaxes:
        rows = c.family == 1
        if c.N < 31 or not bool(rows.any()):
            continue
        y = Q.softmax_model(c.x[rows])
        ref = torch.softmax(c.x[rows].double(), 1)
        sub = ((y > 0) & (y < 2.0 ** -126)).sum(1)
        zero = ((y == 0) & (ref > 0)).sum(1)
        need = 3 if c.N >= 1000 else 1
        assert bool((sub >= need).all()) and bool((zero >= need).all()), c.name


def test_softmax_dominant_rows_peak_in_the_last_stride(softmaxes):
    for c in softmaxes:
        rows = c.family == 5
        if bool(rows.any()):
            assert bool((c.x[rows].argmax(1) == c.N - 1).all())


def test_is_cases(iss):
    """NaN padding; every (N, n) pair with each N meeting all split counts and both ldp; exact zeros, one-hot rows and
    rows that do not sum to 1; a whole-zero column in some one-row split."""
    for c in iss:
        assert bool(torch.isnan(c.pbuf[:, c.N:]).all()) and not bool(torch.isnan(c.p).any())
        assert bool((c.p.sum(1) > 0).all())
    assert {(c.N, c.n) for c in iss} == {(N, n) for N in Q.IS_N for n in Q.IS_ROWS}
    for N in Q.IS_N:
        assert {c.splits for c in iss if c.N == N} == set(Q.IS_SPLITS)
        assert {c.ldp - N for c in iss if c.N == N} == {0, 5}
    big = [c for c in iss if c.N >= 512 and c.n >= 4]
    for c in big:
        p = c.p
        assert bool((p[1::4] == 0).any()) and bool(((p[2::4] == 1).sum(1) == 1).all())
        assert float((p[3::4].double().sum(1) - 1).abs().max()) > 0.05
    assert any(bool((c.p.view(c.splits, c.n, c.N).sum(1) == 0).any()) for c in iss if c.n == 1 and c.N > 1)


# ------------------------------------------------------------------------------------------------ references
def test_ssim_reference_closed_forms(ssim_u8, ssim_f32):
    """Constant pairs equal the closed form, identical pairs give sse 0 and SSIM 1, and the reference's sse is the
    oracle's PSNR arithmetic."""
    t = Q.byte_tables().double()
    for c in ssim_u8[::8] + ssim_f32[::8]:
        sse, ssim = Q.ssim_reference(c)
        va, vb = Q.ssim_values(c)
        for p, k in enumerate(c.kinds):
            if k == "const":
                alpha, beta = float(va[p, 0, 0, 0]), float(vb[p, 0, 0, 0])
                assert abs(float(ssim[p]) - Q.ssim_constant(alpha, beta)) <= Q.ssim_constant_slack(alpha, beta) / 2
            if k == "same":
                assert float(sse[p]) == 0.0 and float(ssim[p]) == 1.0, c.name
            if k in ("noise", "wide"):
                mse = float(sse[p]) / (3 * c.H * c.W)
                want = qo.psnr(va[p].numpy(), vb[p].numpy())
                assert abs(20 * math.log10(1 / math.sqrt(mse)) - want) <= 1e-9
    assert float(t[1, 200]) != float(t[0, 200])


def test_head_reference_against_direct_fp64(heads):
    for c in heads[::9]:
        ref, mag = Q.head_reference(c)
        fa, fb = c.x[:c.P, ..., :c.C].double(), c.x[c.P:, ..., :c.C].double()
        for p in range(c.P):
            acc = 0.0
            for a, b in zip(fa[p].reshape(-1, c.C), fb[p].reshape(-1, c.C)):
                na = a / (math.sqrt(float((a * a).sum())) + 1e-10)
                nb = b / (math.sqrt(float((b * b).sum())) + 1e-10)
                acc += float((c.lin.double() * (na - nb) ** 2).sum())
            assert abs(acc / c.hw - float(ref[p])) <= 1e-13 * float(mag[p]) + 1e-300, c.name
            assert float(ref[p]) <= float(mag[p])
        assert bool((ref[c.equal] == 0).all())


def test_head_bars():
    """Derived roundings stay under the ceiling of the existing head test up to 192 channels and are capped there."""
    assert Q.head_k(32) * Q.U32 < Q.head_k(192) * Q.U32 < Q.HEAD_CEIL < Q.head_k(193) * Q.U32
    assert Q.head_bar(512) == Q.HEAD_CEIL


def test_softmax_reference_on_infinite_rows():
    x = torch.tensor([[0.0, -math.inf, 1.0], [math.inf, 0.0, 1.0], [-math.inf] * 3])
    ref = torch.softmax(x.double(), 1)
    assert float(ref[0, 1]) == 0.0 and bool(torch.isnan(ref[1:]).all())


def test_is_reference_against_scipy_rows(iss):
    from scipy.stats import entropy
    for c in iss[::4]:
        cm, kl = Q.is_reference(c)
        p = c.p.double().numpy().reshape(c.splits, c.n, c.N)
        for k in range(c.splits):
            py = np.mean(p[k], axis=0)
            want = np.mean([entropy(p[k][i], py) for i in range(c.n)])
            assert abs(float(kl[k]) - want) <= 1e-14 * abs(want) + 1e-300
            assert torch.equal(cm[k], torch.from_numpy(py))


# ------------------------------------------------------------------------------------------------ the bars bite
def test_ssim_model_passes_and_mutants_fail(ssim_u8, ssim_f32):
    worst = [0.0, 0.0]
    caught = {m: 0 for m in Q.MUTANTS["ssim"]}
    for c in ssim_u8 + ssim_f32:
        ref = Q.ssim_reference(c)
        ok, es, em, _, msg = Q.ssim_check(c, *Q.ssim_model(c), ref=ref)
        assert ok, msg
        worst = [max(worst[0], es), max(worst[1], em)]
        for m in Q.MUTANTS["ssim"]:
            if m == "ignore_sel_b" and c.form == "f32":
                continue
            ok_m, *_ = Q.ssim_check(c, *Q.ssim_model(c, m), ref=ref)
            assert not ok_m, f"{c.name}: mutant {m} passes"
            caught[m] += 1
    print(f"ssim model: sse rel {worst[0]:.1e}, ssim abs {worst[1]:.1e} (bar {Q.SSIM_BAR:.0e}); mutants caught {caught}")


def test_head_model_passes_and_mutants_fail(heads):
    worst = 0.0
    for c in heads:
        ref = Q.head_reference(c)
        ok, w, msg = Q.head_check(c, Q.head_model(c), ref=ref)
        assert ok, msg
        worst = max(worst, w / Q.head_bar(c.C))
        for m in Q.MUTANTS["head"]:
            targeted = c.hw % Q.HEAD_WARPS != 0 if m == "drop_last" else c.Cs > c.C
            ok_m, *_ = Q.head_check(c, Q.head_model(c, m), ref=ref)
            assert ok_m != targeted, f"{c.name}: mutant {m} {'passes' if ok_m else 'fails an untargeted case'}"
    print(f"head model: worst err / bar {worst:.3f}")


def test_softmax_model_passes_and_mutants_fail(softmaxes):
    """Both mutants fail every 333-row case (all six families); a one-row case may hide them (softmax does not depend
    on the shift, and a last column whose e is 0 adds nothing), but every N still fails through its 333-row cases."""
    worst = 0.0
    for c in softmaxes:
        ok, w, msg = Q.softmax_check(c.x, Q.softmax_model(c.x))
        assert ok, msg
        worst = max(worst, w / Q.softmax_k(c.N))
        for m in Q.MUTANTS["softmax"]:
            ok_m, *_ = Q.softmax_check(c.x, Q.softmax_model(c.x, m))
            assert ok_m == (c.rows == 1 and ok_m), f"{c.name}: mutant {m} passes"
    print(f"softmax model: worst err / bar {worst:.3f}")


def test_is_model_passes_and_mutants_fail(iss):
    """The short column sum fails every case; the NaN zero branch every case whose rows hold an exact zero."""
    for c in iss:
        ref = Q.is_reference(c)
        ok, _, _, msg = Q.is_check(c, *Q.is_model(c), ref=ref)
        assert ok, msg
        for m in Q.MUTANTS["is"]:
            targeted = m == "mean_short" or bool((c.p == 0).any())
            ok_m, *_ = Q.is_check(c, *Q.is_model(c, m), ref=ref)
            assert ok_m != targeted, f"{c.name}: mutant {m} {'passes' if ok_m else 'fails an untargeted case'}"
