"""The exact operands of test_gpu_gemm_fp32_operands.py, checked without a GPU (tests/gemm_fp32_cases.py).

Construction: the kernel's tf32 split of A gives the intended hi and a lo part that is non-zero often in every 64-row
half and k-block, each (64-row half, k-block, 128-column block) of a tile feeds non-zero A_lo.W_hi and A_hi.W_lo products
to some output, every sum stays inside the bit budget, and fp32 computes the reference exactly in two different orders.
Sensitivity: every mutant reference (a fault a kernel could have) moves some output of every case past the check the GPU
test applies, so the GPU test can fail.  Cases are built for an H100 SXM's 132 SMs; the mutant checks run on the first
and the last m block of each case.
"""
import pytest
import torch

from omnitokenizer_b200 import layout as L
from tests import gemm_fp32_cases as FC

S = FC.H100_SMS


def _blocks(M):
    """Logical row slices of the first and the last 128-row m block."""
    last = (M - 1) // 128 * 128
    return [slice(0, min(M, 128))] + ([slice(last, M)] if last > 0 else [])


def _check_split_grid(A):
    hi, lo = FC.split_a(A)
    assert set(hi.unique().tolist()) <= {-1.0, 0.0, 1.0}, "tf32_rn(A) is not the grid's hi"
    assert set((lo / FC.LO_STEP).unique().tolist()) <= {-1.0, 0.0, 1.0}
    assert torch.equal(A - hi, lo) and torch.equal(hi + lo, A)
    assert not ((lo != 0) & (hi == 0)).any(), "lo non-zero where hi is zero"
    return hi, lo


def _lo_density(lo):
    """Fraction of non-zero lo entries in every (64-row half, k-block), rows past M not counted."""
    M, K = lo.shape
    H = -(-M // 64)
    nz = torch.zeros(H * 64, K)
    nz[:M] = (lo != 0).float()
    rows = torch.full((H,), 64.0)
    rows[-1] = M - 64 * (H - 1)
    return nz.view(H, 64, K // FC.KB, FC.KB).sum((1, 3)) / (rows[:, None] * FC.KB)


def _any_per_block(x, size):
    """[rows, K] bool -> [ceil(rows / size), K]: any non-zero in each block of `size` rows."""
    R, K = x.shape
    nb = -(-R // size)
    p = torch.zeros(nb * size, K)
    p[:R] = (x != 0).float()
    return p.view(nb, size, K).amax(1)


def _coverage(a_nz, w_nz, K):
    """[halves, n blocks, k-blocks]: does some row of the half, column of the n block and k of the k-block meet?"""
    kb = K // FC.KB
    return torch.einsum("hbk,nbk->hnb", a_nz.view(-1, kb, FC.KB), w_nz.view(-1, kb, FC.KB)) > 0


def _check_tf32_operands(A, A2, wh, wl, n_split, N):
    """The split grid, lo density, product coverage of every tile and the weight tap cap."""
    K = A.shape[1]
    assert set(wh.unique().tolist()) <= {-1.0, 0.0, 1.0}
    assert set((wl / FC.LO_STEP).unique().tolist()) <= {-1.0, 0.0, 1.0}
    assert not ((wl != 0) & (wh == 0)).any()
    assert int((wh != 0).sum(1).max()) <= FC.MAX_PRODUCTS
    for j, a in enumerate([A] if A2 is None else [A, A2]):
        hi, lo = _check_split_grid(a)
        assert float(_lo_density(lo).min()) >= 0.25, "a (64-row half, k-block) has too few non-zero lo entries"
        cols = slice(0, N) if A2 is None else (slice(0, n_split) if j == 0 else slice(n_split, N))
        for x, w, what in ((lo, wh, "A_lo.W_hi"), (hi, wl, "A_hi.W_lo")):
            w_nz = _any_per_block(w[cols], 128)
            cov = _coverage(_any_per_block(x, 64), w_nz, K)
            assert cov.all(), f"{what}: {int((~cov).sum())} (64-row half, n block, k-block) triples add no product"


def _check_exact(terms_a, terms_w, y, budget):
    """fp64 y = sum of the products; every output's sum of |products| below the budget; fp32 matmuls in two orders
    (k ascending and descending, whatever blocking the CPU library picks) give y exactly."""
    X, Wc = torch.cat(terms_a, 1), torch.cat(terms_w, 1)
    assert torch.equal(X.double() @ Wc.double().t(), y)
    assert float((X.double().abs() @ Wc.double().abs().t()).max()) < budget
    assert torch.equal(y.float().double(), y)
    assert torch.equal((X @ Wc.t()).double(), y)
    assert torch.equal((X.flip(1) @ Wc.flip(1).t()).double(), y)


def _check_tf32_exact(A, wh, wl, y):
    ah, al = FC.split_a(A)
    _check_exact([ah, al, ah], [wh, wh, wl], y, FC.BUDGET)


# ---------------------------------------------------------------- the 3xTF32 tile walk

def test_tf32_round_is_ties_away():
    """The grid's edge cases under the kernel's rule: -1 + 2^-12 is a tie in [1/2, 1) and rounds away to -1."""
    x = torch.tensor([1 + 2.0 ** -12, -1 + 2.0 ** -12, 1 - 2.0 ** -12, -1 - 2.0 ** -12, 2.0 ** -12])
    assert L.tf32_round(x).tolist() == [1.0, -1.0, 1.0, -1.0, 2.0 ** -12]


def test_walk_covers_the_sweep():
    """Every tile count, K, tail and option the sweep promises, and every dual-A split is inside N."""
    assert {c.t for c in FC.TF32_WALK} == set(FC.T_KEYS)
    assert {c.K for c in FC.TF32_WALK} == {32, 64, 1408}
    assert {c.tail for c in FC.TF32_WALK} >= {1, 64, 127}
    plain = [c for c in FC.TF32_WALK if c.epi == "plain"]
    assert any(c.bias for c in plain) and any(c.amap for c in plain) and any(c.cmap for c in plain)
    assert {c.res for c in plain} >= {"sep", "inplace"}
    assert {c.n_split for c in plain} >= {128, 256, 384, 512}
    for i, c in enumerate(FC.TF32_WALK):
        p = FC.walk_problem(c, S, FC.walk_seed(i))
        assert ((p.M + 127) // 128) * ((p.N + 127) // 128) == FC.T_KEYS[c.t](S)
        assert p.n_split < p.N, "dual-A split at or past N"
        if p.amap:
            assert p.amap.seg % 64 == 0 and p.M % p.amap.seg == 0


@pytest.mark.parametrize("i", range(len(FC.TF32_WALK)), ids=[c.id for c in FC.TF32_WALK])
def test_walk_construction(i):
    c = FC.TF32_WALK[i]
    p = FC.walk_problem(c, S, FC.walk_seed(i))
    A, A2 = p.logical()
    _check_tf32_operands(A, A2, p.w_hi, p.w_lo, p.n_split, p.N)
    for t in (p.bias, p.res):
        if t is not None:
            assert float(t.abs().max()) <= 4.0 and torch.equal((t / FC.LO_STEP).round() * FC.LO_STEP, t)
    for rows in _blocks(p.M):
        A, A2 = p.logical(rows)
        y = FC.tf32_y(A, p.w_hi, p.w_lo)
        _check_tf32_exact(A, p.w_hi, p.w_lo, y)
        if A2 is not None:
            _check_tf32_exact(A2, p.w_hi, p.w_lo, FC.tf32_y(A2, p.w_hi, p.w_lo))
        yb = FC.walk_y(p, rows)
        assert torch.equal(yb.float().double(), yb), "y + bias is not exact in fp32"
        out = FC.mutant_output(p, yb, rows)
        assert not FC.walk_fails(p, out, yb, rows), "the true reference fails its own check"


@pytest.mark.parametrize("i", range(len(FC.TF32_WALK)), ids=[c.id for c in FC.TF32_WALK])
def test_walk_mutants_break_every_case(i):
    c = FC.TF32_WALK[i]
    p = FC.walk_problem(c, S, FC.walk_seed(i))
    ys = {str(rows): FC.walk_y(p, rows) for rows in _blocks(p.M)}
    for m in FC.MUTANTS:
        if m == "dual_first" and not p.n_split:
            continue
        caught = False
        for rows in _blocks(p.M):
            ym = FC.walk_y(p, rows, mutant=m)
            caught |= FC.walk_fails(p, FC.mutant_output(p, ym, rows), ys[str(rows)], rows)
        assert caught, f"mutant {m} passes the check of case {c.id}"


# ---------------------------------------------------------------- the 3xTF32 fused QKV epilogue

def _qkv_rows(p):
    """Logical rows [0, r): the first two m blocks (rope positions start at row 0)."""
    return slice(0, min(p.M, 256))


def test_qkv_covers_the_sweep():
    assert {c.tokens for c in FC.TF32_QKV} == {64, 96, 128, 1024}
    assert {c.rope for c in FC.TF32_QKV} == {True, False}
    assert {c.width for c in FC.TF32_QKV if c.width} == set(FC.QKV_WIDTHS)
    for i, c in enumerate(FC.TF32_QKV):
        p = FC.qkv_problem(c, S, FC.qkv_seed(i))
        assert p.M % 128 != 0, "the last m block is full"
        assert p.qk % 128 == 0 and p.qk <= p.N and p.n_split % 128 == 0 and p.n_split < p.N


@pytest.mark.parametrize("i", range(len(FC.TF32_QKV)), ids=[c.id for c in FC.TF32_QKV])
def test_qkv_construction_and_mutants(i):
    c = FC.TF32_QKV[i]
    p = FC.qkv_problem(c, S, FC.qkv_seed(i))
    _check_tf32_operands(p.A, p.A2, p.w_hi, p.w_lo, p.n_split, p.N)
    rows = _qkv_rows(p)
    A, A2 = p.A[rows], None if p.A2 is None else p.A2[rows]
    z = FC.tf32_y(A, p.w_hi, p.w_lo, A2, p.n_split)
    _check_tf32_exact(A, p.w_hi, p.w_lo, FC.tf32_y(A, p.w_hi, p.w_lo))
    assert not FC.qkv_fails(p, torch.cat([FC.qkv_ref(p, z)[0], z[:, p.qk:]], 1), z)
    for m in FC.MUTANTS + ("rope_shift",):
        if (m == "dual_first" and not p.n_split) or (m == "rope_shift" and p.cos is None):
            continue
        if m == "rope_shift":
            got = torch.cat([FC.qkv_ref(p, z, shift_rope=True)[0], z[:, p.qk:]], 1)
        else:
            zm = FC.tf32_y(A, p.w_hi, p.w_lo, A2, p.n_split, mutant=m)
            got = torch.cat([FC.qkv_ref(p, zm)[0], zm[:, p.qk:]], 1)
        assert FC.qkv_fails(p, got, z), f"mutant {m} passes the check of case {c.id}"


# ---------------------------------------------------------------- the CUDA-core fp32 GEMM

def test_fp32_covers_the_sweep():
    cs = FC.FP32_CASES
    assert {c.M for c in cs} >= {1, 127, 128, 129, 4097}
    assert {c.N for c in cs} >= {4, 124, 132, 260, 1536}
    assert {c.K for c in cs} >= {8, 24, 512, 1376}
    assert {c.res for c in cs} >= {"sep", "inplace"} and any(c.bias for c in cs) and any(c.geglu for c in cs)
    assert any(c.n_split for c in cs)
    for c in cs:
        for m in (c.amap, c.cmap):
            if m is not None:
                assert m.seg % 64 != 0 and c.M % m.seg == 0
    assert any(c.amap for c in cs) and any(c.cmap for c in cs)


@pytest.mark.parametrize("i", range(len(FC.FP32_CASES)), ids=[c.id for c in FC.FP32_CASES])
def test_fp32_construction_and_mutants(i):
    c = FC.FP32_CASES[i]
    p = FC.fp32_problem(c, FC.fp32_seed(i))
    assert set((p.W / FC.W_STEP).unique().tolist()) <= {-2.0, -1.0, 0.0, 1.0, 2.0}
    assert int((p.W != 0).sum(1).max()) <= FC.MAX_PRODUCTS
    for a in [p.A] if p.A2 is None else [p.A, p.A2]:
        _check_split_grid(a)
    idx = p.aidx()
    assert int(idx.max()) < p.A.shape[0]
    if c.cmap is not None:
        assert len(set(p.cidx().tolist())) == c.M
    y = FC.fp32_case_y(p)
    for rows in _blocks(c.M):
        A = p.A[idx[rows], : c.K]
        # 2^5: partial sums below it on the 2^-16 grid of the products keep 21 significant bits
        _check_exact([A], [p.W], FC.fp32_y(A, p.W), 2.0 ** 5)
        if p.A2 is not None:
            A2 = p.A2[idx[rows], : c.K]
            _check_exact([A2], [p.W], FC.fp32_y(A2, p.W), 2.0 ** 5)
    assert torch.equal(y.float().double(), y)
    if c.n_split:
        assert not torch.equal(FC.fp32_case_y(p, mutant="dual_first"), y), "dual_first passes"
